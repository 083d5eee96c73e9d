"""GPU: the interaction terms of joint-position control (JointControlSampleModel(characters, interaction_weight,
interaction_margin) with y['scene_placement'] and the reach rows; joint_guidance_step_kernel<true, true, true> in
clusters of C CTAs, DESIGN.md "Joint-position control", "Several characters in one scene").

  1. the guidance iterations alone (b200mdm_test_interaction_guidance) against the fp64 oracle within the bound of
     DESIGN.md, with per-iteration loss, C = 2 and 8, T = 60, HumanML3D and KIT; six mutants miss it 8-fold;
  2. weight 0 without reach rows equals the scene-guided hook and loop bit for bit;
  3. the guided DDPM / DDIM step bit for bit against its tail of hook(denoise(x_t, t)) and its update;
  4. guided loops against the fp32 oracle within 1e-3 on trans_enc, the CLIP decoder and the BERT decoder; a captured
     graph follows a new weight; the interaction adds no launch; scene-aligned shards equal the batch bit for bit;
  5. at B = 64, T = 196, L = 8 the final samples' cross-character joint pairs within r, with the interaction terms
     against joint control alone, reported."""
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import parallel
from b200mdm.engine import interaction_guidance_hook, scene_guidance_hook
from conftest import default_args, rel_err
import interaction_cases as ic
from oracle import dec_emb_oracle as deo
from oracle import interaction_guidance_oracle as io
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ric_oracle
from oracle import schedule_oracle as sch
from test_guided_step_gpu import MODE, _bits_equal, check_update

pytestmark = pytest.mark.gpu
EPS_L = 2.0 ** -16
HOOK_STEP = {2: 3e5, 8: 1e6}   # the hook cases' step in units of 1 / L_GN, as tests/test_interaction_guidance_cpu.py


def _hook(x0, mean, std, inter, lengths, step, K, weight=None):
    B, D, T = x0.shape
    J = jo.n_joints(D)
    pr = inter.pairs if inter.pairs.numel() else None
    return interaction_guidance_hook(x0.cuda(), mean.cuda(), std.cuda(), torch.zeros(B, J, 3, T).cuda(),
                                     torch.zeros(B, J, T).cuda(), step, K, 0.0, 0.0, 0.0, 0.0, 0.0, None, None, inter.C,
                                     inter.weight if weight is None else weight, inter.margin, inter.placement, pr,
                                     inter.reach if pr is not None else None,
                                     inter.pair_weight if pr is not None else None, None, lengths)


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("C", [2, 8])
def test_hook_against_fp64_oracle_and_mutants(D, C):
    T, K = 60, 10
    x0, mean, std, inter, lengths = ic.case(D, T, C, D + C)
    B, J = x0.shape[0], jo.n_joints(D)
    step = ic.step(x0, mean, std, inter) * HOOK_STEP[C]
    got, loss = _hook(x0, mean, std, inter, lengths, step, K)
    got, loss = got.double().cpu(), loss.double().cpu()
    zt, zw = torch.zeros(B, J, 3, T), torch.zeros(B, J, T)
    want, want_loss = io.guide(x0, mean, std, zt, zw, step, K, io.Scene(), inter, None, lengths)
    R = jo.ric_features(J)
    assert torch.equal(got[:, R:], x0[:, R:].double())
    bnd = ic.bound(want, x0, K)
    err = float((got - want).abs().max())
    lerr = float(((loss - want_loss).abs() / (EPS_L * want_loss[0].clamp_min(1e-30))).max())
    print("D %d C %d: |dx| %.3g, err / bound %.3f, loss err / bound %.3f, G %.6g -> %.6g" % (
        D, C, float((want - x0.double()).abs().max()), err / bnd, lerr, float(want_loss[0].sum()),
        float(want_loss[-1].sum())))
    assert err <= bnd and lerr <= 1.0
    for m in io.MUTANTS:
        mut, _ = io.guide_manual(x0, mean, std, zt, zw, step, K, io.Scene(), inter, None, lengths, mutant=m)
        miss = float((got - mut).abs().max()) / bnd
        print("   mutant %-15s misses the bound %.1f-fold" % (m, miss))
        assert miss >= 8.0, m


# ------------------------------------------------------------------------------------------------ steps and loops
STEP, ITERS, CW, FW, FH, LA, RA = 2e-5, 10, 4.0, 2.0, -0.2, 4.0, 0.3


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


def _inter(B, T, C, seed=4):
    """placement of C characters 0.15 m apart per scene, a hand-to-hand and a knee-to-foot row, per-scene weights"""
    _, _, _, inter, _ = ic.case(263, T, C, seed, S=B // C, spacing=0.15)
    return inter


def _y(inp, inter, text=None, **extra):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(),
             text_embed=inp["text_embed"].cuda() if text is None else text, scale=inp["scale"].cuda(),
             scene_placement=inter.placement.float().cuda(), **extra)
    if inter.pairs.numel():
        y.update(interaction_pairs=inter.pairs, interaction_reach=inter.reach.float(),
                 interaction_pair_weight=inter.pair_weight.float().cuda())
    return y


def _jc(cfg, mean, std, C, **kw):
    return b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, **dict(dict(
        contact_weight=CW, floor_weight=FW, floor_height=FH, characters=C, interaction_weight=LA, interaction_margin=RA),
        **kw))


def _loop(diffusion, m, shape, xT, tape, y, sampler="ddpm", eta=0.0, use_graph=True):
    if sampler == "ddpm":
        return diffusion.p_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, use_graph=use_graph,
                                       model_kwargs={"y": y})
    return diffusion.ddim_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, eta=eta, use_graph=use_graph,
                                      model_kwargs={"y": y})


@pytest.fixture(scope="module")
def small():
    B, T, steps, L = 4, 40, 6, 2
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=11, scale=2.5, lengths=[40, 31, 17, 36])
    return B, T, steps, L, cfg, diffusion, sd, inp


def test_zero_weight_is_the_scene_step(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std = jo.motion_stats(263)
    inter = _inter(B, T, 2)._replace(weight=0.0, pairs=torch.zeros(0, 4, dtype=torch.int64))
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    scene = _jc(cfg, mean, std, 1, characters=1, interaction_weight=0.0)
    zero = _jc(cfg, mean, std, 2, interaction_weight=0.0)
    for sampler, eta in (("ddpm", 0.0), ("ddim", 0.5)):
        a = _loop(diffusion, scene, shape, xT, tape, {k: v for k, v in _y(inp, inter).items() if k != "scene_placement"},
                  sampler, eta)
        b = _loop(diffusion, zero, shape, xT, tape, _y(inp, inter), sampler, eta)
        assert torch.equal(a, b), sampler
    x0 = torch.randn(B, 263, T, generator=torch.Generator().manual_seed(2)).cuda()
    J = 22
    args = (x0, mean.cuda(), std.cuda(), torch.zeros(B, J, 3, T).cuda(), torch.zeros(B, J, T).cuda(), STEP, ITERS, CW, FW,
            FH, 0.0, 0.0, None, None)
    h0 = scene_guidance_hook(*args, None, inp["lengths"])
    h1 = interaction_guidance_hook(*args, 2, 0.0, RA, inter.placement, None, None, None, None, inp["lengths"])
    assert torch.equal(h0[0], h1[0]) and torch.equal(h0[1], h1[1])


@pytest.mark.parametrize("sampler,eta,i", [("ddpm", 0.0, 3), ("ddim", 0.5, 4), ("ddim", 0.0, 0)])
def test_guided_step_bit_exact(small, sampler, eta, i):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std = jo.motion_stats(263)
    inter = _inter(B, T, 2)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, 2e-3, ITERS, characters=2, interaction_weight=LA,
                                         interaction_margin=RA)
    y = _y(inp, inter)
    g = torch.Generator().manual_seed(20 + i)
    x_t, noise = torch.randn(B, 263, 1, T, generator=g).cuda(), torch.randn(B, 263, 1, T, generator=g).cuda()
    t = torch.full((B,), i, dtype=torch.long, device="cuda")
    fn = diffusion.p_sample if sampler == "ddpm" else diffusion.ddim_sample
    out = fn(jc, x_t, t, clip_denoised=False, model_kwargs={"y": y}, noise=noise, **({} if sampler == "ddpm" else {"eta": eta}))
    x0 = jc(x_t, t, y=_y(inp, inter))                                        # the plain model's x0
    h, _ = interaction_guidance_hook(x0.reshape(B, 263, T), mean.cuda(), std.cuda(), torch.zeros(B, 22, 3, T).cuda(),
                                     torch.zeros(B, 22, T).cuda(), 2e-3, ITERS, 0.0, 0.0, 0.0, 0.0, 0.0, None, None, 2, LA,
                                     RA, inter.placement, inter.pairs, inter.reach, inter.pair_weight, None, inp["lengths"])
    pred = h.reshape(x0.shape)
    moved = float((pred - x0).abs().max())
    print("%s eta %.1f i %d: guidance moves x0 by %.3g; pred_xstart == hook(denoise) %s"
          % (sampler, eta, i, moved, _bits_equal(pred, out["pred_xstart"])))
    assert moved > 1e-3 and _bits_equal(pred, out["pred_xstart"])
    check_update(MODE[sampler], diffusion.schedule_rows(eta)[i], pred, x_t, noise, out["sample"], i)


def _control(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    mean, std = jo.motion_stats(263)
    x = torch.randn(B, 263, T, generator=g) * 0.5
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    target = ric_oracle.recover_from_ric(data, 22).permute(0, 2, 3, 1).float()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    return mean, std, target, weight


def _oracle_loop(den, control, inter, lengths, tabs, tape, sampler="ddpm", eta=0.0):
    mean, std, target, weight = control
    f = io.guided_denoiser(den, mean, std, target, weight, STEP, ITERS, io.Scene(CW, FW, FH), inter, None, lengths)
    with torch.no_grad():
        return deo.sample_loop(f, tabs, tape, sampler=sampler, eta=eta)


def test_loops_against_oracle_graph_and_launches(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    control = _control(B, T, 5)
    mean, std, target, weight = control
    inter = _inter(B, T, 2)
    jc = _jc(cfg, mean, std, 2)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    den = po.enc_denoiser(mo.OracleWeights(sd, L), list(range(steps)), inp["text_embed"], inp["scale"], inp["lengths"])
    tabs = sch.diffusion_tables(sch.named_betas("cosine", steps))
    for sampler, eta in (("ddpm", 0.0), ("ddim", 0.0), ("ddim", 0.5)):
        out = _loop(diffusion, jc, shape, xT, tape, _y(inp, inter, **joint), sampler, eta)
        ref = _oracle_loop(den, control, inter, inp["lengths"], tabs, inp["tape"], sampler, eta)
        e = rel_err(out, ref)
        print("trans_enc, C 2, %s eta %.1f: engine vs oracle %.2e" % (sampler, eta, e))
        assert e < 1e-3
    y = _y(inp, inter, **joint)
    prog = list(diffusion.p_sample_loop_progressive(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape,
                                                    model_kwargs={"y": y}))
    assert torch.equal(prog[-1]["sample"], _loop(diffusion, jc, shape, xT, tape, y))
    # a new weight reaches the captured step graph (same key: no recapture), and the interaction adds no launch
    eng = cfg.model.engine()
    jc8 = _jc(cfg, mean, std, 2, interaction_weight=2 * LA)
    torch.cuda.synchronize()
    eng.launch_count(reset=True)
    a = _loop(diffusion, jc8, shape, xT, tape, y)
    torch.cuda.synchronize()
    n_inter = eng.launch_count()
    assert torch.equal(a, _loop(diffusion, jc8, shape, xT, tape, y, use_graph=False)) and not torch.equal(a, prog[-1]["sample"])
    scene = _jc(cfg, mean, std, 1, characters=1, interaction_weight=0.0)
    torch.cuda.synchronize()
    eng.launch_count(reset=True)
    _loop(diffusion, scene, shape, xT, tape, {k: v for k, v in y.items() if k in ("mask", "lengths", "text_embed", "scale",
                                                                                  "joint_target", "joint_weight")})
    torch.cuda.synchronize()
    print("launches of a %d-step loop: scene-guided %d, with interaction %d" % (steps, eng.launch_count(), n_inter))
    assert eng.launch_count() == n_inter
    # scene-aligned shards equal the batch
    kw = {"y": y}
    full = diffusion.p_sample_loop(jc, shape, clip_denoised=False, model_kwargs=kw, noise_seed=9)
    parts = [diffusion.p_sample_loop(jc, (hi - lo,) + shape[1:], clip_denoised=False, noise_seed=9, sample_index_base=lo,
                                     model_kwargs=parallel.shard_model_kwargs(kw, lo, hi, characters=2))
             for lo, hi in ((0, 2), (2, 4))]
    assert torch.equal(torch.cat(parts), full)


@pytest.mark.parametrize("memory", ["clip", "bert"])
def test_decoders_against_oracle(memory):
    B, T, steps, L = 4, 40, 6, 2
    cfg, diffusion, sd = _dec(L, steps, memory)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=12, scale=2.5, lengths=[40, 33, 20, 38])
    control = _control(B, T, 9)
    mean, std, target, weight = control
    inter = _inter(B, T, 2, seed=6)
    jc = _jc(cfg, mean, std, 2)
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
    for sampler, eta in (("ddpm", 0.0), ("ddim", 0.5)):
        y = _y(inp, inter, text, joint_target=target.cuda(), joint_weight=weight.cuda())
        out = _loop(diffusion, jc, (B, 263, 1, T), xT, tape, y, sampler, eta)
        ref = _oracle_loop(den, control, inter, inp["lengths"], tabs, inp["tape"], sampler, eta)
        e = rel_err(out, ref)
        print("%s decoder, C 2, %s eta %.1f: engine vs oracle %.2e" % (memory, sampler, eta, e))
        assert e < 1e-3


def close_pairs(sample, mean, std, placement, C, lengths, r=RA):
    """cross-character joint pairs (j, k) within r of each other in the scene frame, summed over frames t < L_ab"""
    xyz = ric_oracle.sample_to_xyz(sample.cpu(), mean, std).double().permute(0, 3, 1, 2)     # [B, T, J, 3]
    B, T, J, _ = xyz.shape
    Q = io.place(xyz, placement.cpu()).reshape(B // C, C, T, J, 3)
    L = lengths.cpu().reshape(B // C, C)
    n = 0
    for a in range(C):
        for b in range(a + 1, C):
            live = torch.arange(T)[None, :] < torch.minimum(L[:, a], L[:, b])[:, None]
            d = (Q[:, a, :, :, None] - Q[:, b, :, None, :]).pow(2).sum(-1).sqrt()
            n += int(((d < r) & live[:, :, None, None]).sum())
    return n


def test_headline_b64_effect():
    B, T, steps, L, C = 64, 196, 50, 8, 2
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=2.5)
    mean, std = jo.motion_stats(263)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    # two characters 0.4 m apart facing each other; pelvis targets walk each through the other's start
    pl = torch.zeros(B, 3)
    pl[1::2, 0], pl[1::2, 2] = 0.4, torch.pi
    s = torch.linspace(0.0, 0.4, T)
    target = torch.zeros(B, 22, 3, T)
    target[:, 0, 0], target[:, 0, 1] = s, 0.9
    weight = torch.zeros(B, 22, T)
    weight[:, 0, ::4] = 1.0
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
                scale=inp["scale"].cuda(), **joint)
    plain_jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    plain = _loop(diffusion, plain_jc, shape, xT, tape, base)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, characters=C, interaction_weight=LA,
                                         interaction_margin=RA)
    out = _loop(diffusion, jc, shape, xT, tape, dict(base, scene_placement=pl.cuda()))
    assert bool(torch.isfinite(out).all()) and not torch.equal(out, plain)
    ng = close_pairs(out, mean, std, pl, C, inp["lengths"])
    nu = close_pairs(plain, mean, std, pl, C, inp["lengths"])
    print("enc B=64 T=196 L=8 DDPM 50, C %d, K %d, lambda %.0e, la %.1f, r %.1f, pelvis targets crossing: joint pairs "
          "within r guided %d, joint control alone %d (ratio %.4f)" % (C, ITERS, STEP, LA, RA, ng, nu, ng / max(nu, 1)))
