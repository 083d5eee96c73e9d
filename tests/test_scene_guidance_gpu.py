"""GPU: the scene terms of joint-position control (JointControlSampleModel(obstacle_weight, obstacle_margin) with
y['obstacle_sdf'] / y['terrain']; joint_guidance_step_kernel<true, true>, DESIGN.md "Joint-position control", "Scene:
obstacles and uneven ground").

  1. the guidance iterations alone (b200mdm_test_scene_guidance) against the fp64 oracle within the bound of DESIGN.md,
     HumanML3D and KIT, T = 2, 60, 196, at lambda = 1 / L_GN: per-sample planar grids over 10 iterations (scene terms
     alone, and with joint and contact terms), curved grids over one iteration with every active joint >= 1e-3 cell from
     a grid line (T <= 60); six mutants miss it 8-fold with the scene terms alone at T = 60; the total G never
     increases;
  2. an all-zero terrain is the flat floor bit for bit, an SDF >= r everywhere is the scene-free loop bit for bit, the
     scene adds no launch, and the unguided step graph is unchanged after it; the C ABI's state checks;
  3. guided loops against the fp32 oracle within 1e-3 at lambda = 2e-4 (DDPM, DDIM eta 0 and 0.5, the single-step and
     progressive forms), shared and per-sample planar grids, on trans_enc, the CLIP decoder with a timestep token and the
     BERT decoder; Philox shards with per-sample grids equal the batch bit for bit;
  4. at B = 64, T = 196, L = 8 the final samples' obstacle and terrain penetration (through sample_to_xyz) against
     unguided samples on the same noise, reported."""
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from b200mdm.engine import foot_guidance_hook, scene_guidance_hook
from conftest import default_args, rel_err
import scene_cases as sc
from oracle import dec_emb_oracle as deo
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ric_oracle
from oracle import scene_guidance_oracle as so
from oracle import schedule_oracle as sch

pytestmark = pytest.mark.gpu
RTOL = 1e-3
U32 = 2.0 ** -24
EPS_G = 2.0 ** -12
EPS_L = 2.0 ** -16


def _extent(x0, mean, std, target):
    p0 = ric_oracle.recover_from_ric((x0.double() * std.double()[None, :, None] + mean.double()[None, :, None])
                                     .permute(0, 2, 1), jo.n_joints(x0.shape[1]))
    return float(p0[..., [0, 2]].max() - p0[..., [0, 2]].min()) + float(target[:, :, [0, 2]].abs().max()) + 1.0


def _check_hook(x0, mean, std, target, weight, lengths, sdf, terrain, cw, K, label, mutants=False, fh=sc.FH):
    T = x0.shape[-1]
    step = so.step_bound(std, weight, _extent(x0, mean, std, target), T, cw, sc.FW, sc.OW, sdf, terrain)
    terms = (cw, sc.FW, fh, sc.OW, sc.R, sdf, terrain, None, lengths)
    got, loss = scene_guidance_hook(x0.cuda(), mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), step, K, cw, sc.FW,
                                    fh, sc.OW, sc.R, sdf, terrain, None, lengths)
    got, loss = got.double().cpu(), loss.double().cpu()
    want, want_loss = so.guide(x0, mean, std, target, weight, step, K, *terms)
    R = jo.ric_features(jo.n_joints(x0.shape[1]))
    assert torch.equal(got[:, R:], x0[:, R:].double())
    disp = float((want - x0.double()).abs().max())
    bound = EPS_G * disp + 2 * U32 * K * float(x0.abs().max())
    err = float((got - want).abs().max())
    lerr = float(((loss - want_loss).abs() / (EPS_L * want_loss[0].clamp_min(1e-30))).max())
    print("%s K %2d step %.3g: |dx| %.2e, err / bound %.3f, loss err / bound %.3f, G %.5g -> %.5g"
          % (label, K, step, disp, err / bound, lerr, float(want_loss[0].sum()), float(want_loss[-1].sum())))
    assert err <= bound and lerr <= 1.0, label
    assert bool((loss[1:] <= loss[:-1] * (1 + 1e-6)).all()), label
    if mutants:
        for m in so.MUTANTS:
            mut, _ = so.guide_manual(x0, mean, std, target, weight, step, K, *terms, mutant=m)
            miss = float((got - mut.double()).abs().max()) / bound
            print("   mutant %-14s misses the bound %.1f-fold" % (m, miss))
            assert miss >= 8.0, (label, m, miss)


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [2, 60, 196])
def test_hook_against_fp64_oracle_and_mutants(D, T):
    x0, mean, std, target, weight, lengths, sdf, terrain = sc.planar_case(D, T, seed=D * 1000 + T, B=3)
    x0, target = x0.float(), target.float()
    # the scene terms alone, on motions that stay near the grids (|x0| <= ~1.3) and a floor at 0.2 m that most joints
    # meet: the iterations move x0 well above the bound's rounding floor, so each mutant's miss shows
    _check_hook(x0 * (0.3 / 0.7), mean, std, torch.zeros_like(target), weight, lengths, sdf, terrain, 0.0, 10,
                "D %d T %3d planar, scene only" % (D, T), mutants=T == 60, fh=0.2)
    g = torch.Generator().manual_seed(T)
    weight = (torch.rand(weight.shape, generator=g) < 0.2).float()
    _check_hook(x0, mean, std, target, weight, lengths, sdf, terrain, sc.CW, 10, "D %d T %3d planar, joint + foot" % (D, T))
    if T > 60:   # (longer motions have too many active joints to keep all of them clear of the grid lines)
        return
    x0, mean, std, target, weight, lengths, sdf, terrain, n_o, n_f = sc.curved_case(D, T, seed=D + T)
    _check_hook(x0.float(), mean, std, target.float(), weight.float(), lengths, sdf, terrain, sc.CW, 1,
                "D %d T %3d curved (%d / %d active joints)" % (D, T, n_o, n_f))


# ------------------------------------------------------------------------------------------------ loops
STEP, ITERS, CW, FW, FH, OW, R = 2e-4, 10, 4.0, 2.0, -0.2, 4.0, 0.3


def _enc(layers, steps, seed=1):
    args = default_args(layers=layers, diffusion_steps=steps)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=layers, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), diffusion, sd


def _dec(layers, steps, memory, seed=0):
    bert = memory == "bert"
    args = default_args(layers=layers, diffusion_steps=steps, arch="trans_dec", text_encoder_type=memory,
                        emb_trans_dec=not bert)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=layers, cond_dim=768 if bert else 512, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), diffusion, sd


def _control(B, T, seed):
    """targets: the pelvis of a random normalised motion on every frame"""
    g = torch.Generator().manual_seed(seed)
    mean, std = jo.motion_stats(263)
    x = torch.randn(B, 263, T, generator=g) * 0.5
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    target = ric_oracle.recover_from_ric(data, 22).permute(0, 2, 3, 1).float()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    return mean, std, target, weight


def _grids(B, per_sample):
    """planar obstacle SDF and terrain over [-2, 1.25] x [-1.5, 1.25], per sample or sample 0's shared"""
    o, c = (-2.0, -1.5), 0.25
    sdf = sc._planar(B, 12, 14, o, c, [(0.3, 0.8, -0.5), (0.1, -0.6, 0.7), (0.2, 0.5, 0.5)] * B)
    ter = sc._planar(B, 12, 14, o, c, [(0.05, 0.3, 0.2), (-0.1, -0.2, 0.4), (0.0, 0.25, -0.3)] * B)
    if not per_sample:
        sdf, ter = sdf[0], ter[0]
    return b200mdm.SceneGrid(sdf, o, c), b200mdm.SceneGrid(ter, o, c)


def _pick(grid, idx):
    return b200mdm.SceneGrid(grid.values[idx], grid.origin, grid.cell) if grid.per_sample else grid


def _y(inp, text=None, **extra):
    return dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(),
                text_embed=inp["text_embed"].cuda() if text is None else text, scale=inp["scale"].cuda(), **extra)


def _loop(diffusion, m, shape, xT, tape, y, sampler="ddpm", eta=0.0, use_graph=True):
    if sampler == "ddpm":
        return diffusion.p_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, use_graph=use_graph,
                                       model_kwargs={"y": y})
    return diffusion.ddim_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, eta=eta, use_graph=use_graph,
                                      model_kwargs={"y": y})


def _jc(cfg, mean, std, **kw):
    return b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, **dict(dict(contact_weight=CW, floor_weight=FW,
                                                                                   floor_height=FH), **kw))


@pytest.fixture(scope="module")
def small():
    B, T, steps, L = 3, 40, 6, 2
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=11, scale=2.5, lengths=[40, 31, 17])
    return B, T, steps, L, cfg, diffusion, sd, inp


def test_identities_kernel_count_and_state(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 3)
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    foot = _jc(cfg, mean, std)
    scene = _jc(cfg, mean, std, obstacle_weight=OW, obstacle_margin=R)
    sdf, ter = _grids(B, True)
    flat = b200mdm.SceneGrid(torch.zeros(B, 5, 7), (-1.0, -1.0), 0.5)
    far = b200mdm.SceneGrid(torch.full((6, 6), R + 1.0), (-1.0, -1.0), 0.5)
    for use_graph in (True, False):
        for sampler in ("ddpm", "ddim"):
            a = _loop(diffusion, foot, shape, xT, tape, _y(inp, **joint), sampler, 0.0, use_graph)
            b = _loop(diffusion, foot, shape, xT, tape, _y(inp, terrain=flat, **joint), sampler, 0.0, use_graph)
            c = _loop(diffusion, scene, shape, xT, tape, _y(inp, obstacle_sdf=far, **joint), sampler, 0.0, use_graph)
            d = _loop(diffusion, scene, shape, xT, tape, _y(inp, obstacle_sdf=sdf, terrain=ter, **joint), sampler, 0.0, use_graph)
            assert torch.equal(a, b) and torch.equal(a, c), (use_graph, sampler)
            assert not torch.equal(a, d)
    # the hook: the same identities on one x0
    x0 = torch.randn(B, 263, T, generator=torch.Generator().manual_seed(2)).cuda()
    args = (x0, mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, ITERS, CW, FW, FH)
    h0 = foot_guidance_hook(*args, None, inp["lengths"])
    for grids in ((None, flat), (far, None), (far, flat)):
        h1 = scene_guidance_hook(*args, OW if grids[0] is not None else 0.0, R, *grids, None, inp["lengths"])
        assert torch.equal(h0[0], h1[0]) and torch.equal(h0[1], h1[1]), grids
    # one launch count with or without the scene
    eng = cfg.model.engine()
    counts = {}
    for name, m, extra in (("foot", foot, {}), ("scene", scene, dict(obstacle_sdf=sdf, terrain=ter))):
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        _loop(diffusion, m, shape, xT, tape, _y(inp, **extra, **joint))
        torch.cuda.synchronize()
        counts[name] = eng.launch_count()
    print("launches of a %d-step loop: joint + foot %d, joint + foot + scene %d" % (steps, counts["foot"], counts["scene"]))
    assert counts["foot"] == counts["scene"]
    # the unguided step graph, and joint + foot, after a scene loop equal a fresh engine's
    after = _loop(diffusion, cfg, shape, xT, tape, _y(inp))
    with pytest.raises(_lib.B200MDMError) as ex:     # no joint guidance for the current conditioning
        eng.set_scene_guidance(OW, R, sdf)
    assert ex.value.code == _lib.ESTATE
    fresh, _, _ = _enc(L, steps)
    want = _loop(diffusion, fresh, shape, xT, tape, _y(inp))
    fresh.model.engine().close()
    assert torch.equal(after, want)
    foot_alone = _loop(diffusion, foot, shape, xT, tape, _y(inp, **joint))
    _loop(diffusion, scene, shape, xT, tape, _y(inp, obstacle_sdf=sdf, terrain=ter, **joint))
    assert torch.equal(_loop(diffusion, foot, shape, xT, tape, _y(inp, **joint)), foot_alone)


def _oracle_loop(den, control, idx, sdf, ter, lengths, tabs, tape, sampler="ddpm", eta=0.0):
    mean, std, target, weight = control
    f = so.guided_denoiser(den, mean, std, target[idx], weight[idx], STEP, ITERS, CW, FW, FH, OW, R, _pick(sdf, idx),
                           _pick(ter, idx), None, lengths[idx])
    with torch.no_grad():
        return deo.sample_loop(f, tabs, [t[idx] for t in tape], sampler=sampler, eta=eta)


def test_guided_loops_against_oracle_small(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    control = _control(B, T, 5)
    mean, std, target, weight = control
    jc = _jc(cfg, mean, std, obstacle_weight=OW, obstacle_margin=R)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    idx = list(range(B))
    den = po.enc_denoiser(mo.OracleWeights(sd, L), list(range(steps)), inp["text_embed"], inp["scale"], inp["lengths"])
    tabs = sch.diffusion_tables(sch.named_betas("cosine", steps))
    for per_sample in (False, True):
        sdf, ter = _grids(B, per_sample)
        for sampler, eta in (("ddpm", 0.0), ("ddim", 0.0), ("ddim", 0.5)):
            out = _loop(diffusion, jc, shape, xT, tape, _y(inp, obstacle_sdf=sdf, terrain=ter, **joint), sampler, eta)
            ref = _oracle_loop(den, control, idx, sdf, ter, inp["lengths"], tabs, inp["tape"], sampler, eta)
            e = rel_err(out, ref)
            print("trans_enc, per-sample grids %d, %s eta %.1f: engine vs oracle %.2e" % (per_sample, sampler, eta, e))
            assert e < RTOL
    y = _y(inp, obstacle_sdf=sdf, terrain=ter, **joint)
    prog = list(diffusion.p_sample_loop_progressive(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape,
                                                    model_kwargs={"y": y}))
    loop = _loop(diffusion, jc, shape, xT, tape, y)
    assert torch.equal(prog[-1]["sample"], loop)
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    one = diffusion.p_sample(jc, prog[-2]["sample"], t, clip_denoised=False, model_kwargs={"y": y}, noise=tape[-1])
    assert torch.equal(one["sample"], loop)
    dprog = list(diffusion.ddim_sample_loop_progressive(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape, eta=0.5,
                                                        model_kwargs={"y": y}))
    assert torch.equal(dprog[-1]["sample"], _loop(diffusion, jc, shape, xT, tape, y, "ddim", 0.5))
    # scene terms without joint keys, contact or floor weight: the obstacles alone
    alone = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, obstacle_weight=OW, obstacle_margin=R)
    out = _loop(diffusion, alone, shape, xT, tape, _y(inp, obstacle_sdf=sdf))
    f = so.guided_denoiser(den, mean, std, target, torch.zeros_like(weight), STEP, ITERS, 0.0, 0.0, 0.0, OW, R, sdf, None,
                           None, inp["lengths"])
    with torch.no_grad():
        ref = deo.sample_loop(f, tabs, inp["tape"])
    e = rel_err(out, ref)
    print("trans_enc, obstacles alone: engine vs oracle %.2e" % e)
    assert e < RTOL


def test_sharding_with_per_sample_grids(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 8)
    jc = _jc(cfg, mean, std, obstacle_weight=OW, obstacle_margin=R)
    sdf, ter = _grids(B, True)
    shape = (B, 263, 1, T)
    kw = {"y": _y(inp, obstacle_sdf=sdf, terrain=ter, joint_target=target.cuda(), joint_weight=weight.cuda())}
    full = diffusion.p_sample_loop(jc, shape, clip_denoised=False, model_kwargs=kw, noise_seed=9)
    parts = []
    for lo, hi in ((0, 1), (1, 3)):
        parts.append(diffusion.p_sample_loop(jc, (hi - lo,) + shape[1:], clip_denoised=False, noise_seed=9, sample_index_base=lo,
                                             model_kwargs=parallel.shard_model_kwargs(kw, lo, hi)))
    assert torch.equal(torch.cat(parts), full)


@pytest.mark.parametrize("memory", ["clip", "bert"])
def test_decoders_against_oracle(memory):
    B, T, steps, L = 3, 40, 6, 2
    cfg, diffusion, sd = _dec(L, steps, memory)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=12, scale=2.5, lengths=[40, 33, 20])
    control = _control(B, T, 9)
    mean, std, target, weight = control
    jc = _jc(cfg, mean, std, obstacle_weight=OW, obstacle_margin=R)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    W = mo.OracleWeights(sd, L)
    if memory == "bert":
        enc, tmask, _ = b200mdm.synthetic_dip_inputs(B, 20, 0, seed=13)
        tmask[:] = False
        tmask[1, 14:] = True
        text = (enc.cuda(), tmask.cuda())
        no_prefix = lambda x: x.new_zeros(x.shape[:-1] + (0,))   # noqa: E731
        den = lambda x, i: mo.cfg_denoise_dec(W, x, i, enc, tmask, no_prefix(x), inp["scale"], inp["lengths"])   # noqa: E731
    else:
        text = None
        den = deo.denoiser(W, list(range(steps)), inp["text_embed"], inp["scale"], inp["lengths"])
    tabs = sch.diffusion_tables(sch.named_betas("cosine", steps))
    for per_sample, sampler, eta in ((True, "ddpm", 0.0), (False, "ddim", 0.5)):
        sdf, ter = _grids(B, per_sample)
        y = _y(inp, text, obstacle_sdf=sdf, terrain=ter, joint_target=target.cuda(), joint_weight=weight.cuda())
        out = _loop(diffusion, jc, (B, 263, 1, T), xT, tape, y, sampler, eta)
        ref = _oracle_loop(den, control, list(range(B)), sdf, ter, inp["lengths"], tabs, inp["tape"], sampler, eta)
        e = rel_err(out, ref)
        print("%s decoder, per-sample grids %d, %s eta %.1f: engine vs oracle %.2e" % (memory, per_sample, sampler, eta, e))
        assert e < RTOL


def _penetration(sample, mean, std, discs, boxes, slope, lengths):
    """(obstacle penetration sum max(R - sdf, 0), terrain penetration sum max(FH + H - y, 0)) in metres over the joints
    and frames t < lengths[b] of the samples (sample_to_xyz), with the exact SDF of the shapes and the planar terrain"""
    xyz = ric_oracle.sample_to_xyz(sample.cpu(), mean, std).double()               # [B, J, 3, T]
    live = (torch.arange(xyz.shape[-1])[None, :] < lengths.cpu()[:, None])[:, None]
    x, y, z = xyz[:, :, 0], xyz[:, :, 1], xyz[:, :, 2]
    S = torch.from_numpy(b200mdm.shape_sdf(x.numpy(), z.numpy(), discs, boxes))
    H = slope[0] + slope[1] * x + slope[2] * z
    return float(((R - S).clamp_min(0) * live).sum()), float(((FH + H - y).clamp_min(0) * live).sum())


def test_headline_b64_effect():
    B, T, steps, L = 64, 196, 50, 8
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=2.5)
    mean, std = jo.motion_stats(263)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    plain = _loop(diffusion, cfg, shape, xT, tape, _y(inp))
    # obstacles where the unguided motions go: discs and a wall box around their mean root path
    xyz = ric_oracle.sample_to_xyz(plain.cpu(), mean, std).double()
    cx, cz = float(xyz[:, 0, 0].mean()), float(xyz[:, 0, 2].mean())
    discs = [(cx, cz, 0.4), (cx + 1.0, cz + 0.5, 0.3), (cx - 0.8, cz - 0.6, 0.3)]
    boxes = [(cx - 2.0, cz + 1.0, cx + 2.0, cz + 1.2)]
    o, c = (cx - 4.0, cz - 4.0), 0.05
    sdf = b200mdm.SceneGrid.from_shapes((161, 161), o, c, discs, boxes)
    slope = (0.0, 0.1, -0.05)
    zz = o[1] + c * torch.arange(161, dtype=torch.float64)[:, None]
    xx = o[0] + c * torch.arange(161, dtype=torch.float64)[None, :]
    ter = b200mdm.SceneGrid(slope[0] + slope[1] * xx + slope[2] * zz, o, c)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, floor_weight=FW, floor_height=FH, obstacle_weight=OW,
                                         obstacle_margin=R)
    out = _loop(diffusion, jc, shape, xT, tape, _y(inp, obstacle_sdf=sdf, terrain=ter))
    assert bool(torch.isfinite(out).all()) and not torch.equal(out, plain)
    og, tg = _penetration(out, mean, std, discs, boxes, slope, inp["lengths"])
    op, tp = _penetration(plain, mean, std, discs, boxes, slope, inp["lengths"])
    print("enc B=64 T=196 L=8 DDPM 50, K %d, lambda %.0e, lo %.1f, r %.1f, lf %.1f: obstacle penetration guided %.5g m, "
          "unguided %.5g m (ratio %.4f); terrain penetration guided %.5g m, unguided %.5g m (ratio %.4f)"
          % (ITERS, STEP, OW, R, FW, og, op, og / max(op, 1e-30), tg, tp, tg / max(tp, 1e-30)))
