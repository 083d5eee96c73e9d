"""GPU: the foot-contact and floor terms of joint-position control (JointControlSampleModel(contact_weight, floor_weight,
floor_height); joint_guidance_step_kernel<true>, DESIGN.md "Joint-position control", "Foot contact and floor").

  1. the guidance iterations alone (b200mdm_test_foot_guidance) against the fp64 oracle within the bound of DESIGN.md,
     HumanML3D and KIT, T = 1, 2, 60, 196, 256, derived and given contacts, with and without joint terms and lengths;
     five mutants (kappa on the pair (t-1, t), left / right swapped, Delta's sign, max for min, lengths ignored) miss it
     8-fold with the foot terms alone; the total G never increases;
  2. zero foot weights are the plain joint-controlled loop bit for bit, a y['foot_contact'] equal to the derived mask is
     the derived loop bit for bit, and a guided step with the foot terms launches as many kernels as one without;
  3. guided loops against the fp32 oracle within 1e-3: DDPM, DDIM eta 0 and 0.5, inpainting, the single-step and
     progressive forms, joint + foot and foot only, the encoder and the CLIP decoder with a timestep token; B = 64,
     T = 196, L = 8 for the encoder, where the contact energy of the final samples (their own contacts, through
     sample_to_xyz) falls with guidance;
  4. the sampler's set_cond drops the foot terms; Philox shards equal the batch bit for bit."""
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import parallel
from b200mdm.engine import foot_guidance_hook
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import foot_guidance_oracle as fo
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ric_oracle
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
U32 = 2.0 ** -24
EPS_G = 2.0 ** -12
EPS_L = 2.0 ** -16


def _positions(x, mean, std):
    D = x.shape[1]
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    return ric_oracle.recover_from_ric(data, jo.n_joints(D)).permute(0, 2, 3, 1)


def _hook_case(D, T, seed, joint=True, given=False):
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    B = 3
    x0 = (torch.randn(B, D, T, generator=g) * 0.7).float()
    target = _positions(torch.randn(B, D, T, generator=g) * 0.7, mean, std).float()
    weight = torch.zeros(B, J, T)
    if joint:
        weight[:, 0] = 1.0
        for j in (20, 21) if J == 22 else (4, 7):
            weight[:, j, torch.randint(0, T, (max(1, T // 20),), generator=g)] = 1.0
    contact = torch.rand(B, 4, T, generator=g) * (torch.rand(B, 4, T, generator=g) < 0.5) if given else None
    lengths = torch.tensor([T, max(1, T - 9), max(1, T // 2)])
    p0 = _positions(x0, mean, std)
    extent = float(p0[:, :, [0, 2]].max() - p0[:, :, [0, 2]].min()) + float(target[:, :, [0, 2]].abs().max()) + 1.0
    return x0, mean, std, target, weight, contact, lengths, extent


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [1, 2, 60, 196, 256])
def test_hook_against_fp64_oracle_and_mutants(D, T):
    cw, fw, fh = 4.0, 2.0, 0.0
    for joint, given, K in ((True, False, 10), (False, False, 10), (True, True, 1), (False, True, 10)):
        x0, mean, std, target, weight, contact, lengths, extent = _hook_case(D, T, D * 1000 + T + K, joint, given)
        kmax = 1.0 if contact is None else float(contact.max())
        step = fo.step_bound(std, weight, extent, T, cw, fw, kmax)
        got, loss = foot_guidance_hook(x0.cuda(), mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), step, K, cw, fw, fh,
                                       None if contact is None else contact.cuda(), lengths)
        got, loss = got.double().cpu(), loss.double().cpu()
        want, want_loss = fo.guide(x0, mean, std, target, weight, step, K, cw, fw, fh, contact, lengths)
        R = jo.ric_features(jo.n_joints(D))
        assert torch.equal(got[:, R:], x0[:, R:].double())
        disp = float((want - x0.double()).abs().max())
        bound = EPS_G * disp + 2 * U32 * K * float(x0.abs().max())
        err = float((got - want).abs().max())
        lerr = float(((loss - want_loss).abs() / (EPS_L * want_loss[0].clamp_min(1e-30))).max())
        print("D %d T %3d joint %d given %d K %2d: |dx| %.2e, err / bound %.3f, loss err / bound %.3f, G %.4g -> %.4g"
              % (D, T, joint, given, K, disp, err / bound, lerr, float(want_loss[0].sum()), float(want_loss[-1].sum())))
        assert err <= bound and lerr <= 1.0, (joint, given, K)
        assert bool((loss[1:] <= loss[:-1] * (1 + 1e-6)).all()), (joint, given, K)
        if T >= 60 and not joint:   # with joint terms on every frame the step bound leaves the foot terms little pull
            for m in fo.MUTANTS:
                mut, _ = fo.guide_manual(x0, mean, std, target, weight, step, K, cw, fw, fh, contact, lengths, mutant=m)
                miss = float((got - mut.double()).abs().max()) / bound
                print("   mutant %-11s misses the bound %.1f-fold" % (m, miss))
                assert miss >= 8.0, (joint, given, K, m, miss)


# ------------------------------------------------------------------------------------------------ loops
def _enc(layers, steps, seed=1):
    args = default_args(layers=layers, diffusion_steps=steps)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=layers, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), diffusion, sd


def _dec(layers, steps, seed=0):
    args = default_args(layers=layers, diffusion_steps=steps, arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=layers, cond_dim=512, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), diffusion, sd


def _control(B, T, seed):
    """targets: the pelvis of a random normalised motion on every frame"""
    g = torch.Generator().manual_seed(seed)
    mean, std = jo.motion_stats(263)
    target = _positions(torch.randn(B, 263, T, generator=g) * 0.5, mean, std).float()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    return mean, std, target, weight


def _y(inp, **extra):
    return dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
                scale=inp["scale"].cuda(), **extra)


STEP, ITERS, CW, FW, FH = 2e-4, 10, 4.0, 2.0, 0.0


@pytest.fixture(scope="module")
def small():
    B, T, steps, L = 3, 40, 6, 2
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=11, scale=2.5, lengths=[40, 31, 17])
    return B, T, steps, L, cfg, diffusion, sd, inp


def _loop(diffusion, m, shape, xT, tape, y, sampler="ddpm", eta=0.0, use_graph=True):
    if sampler == "ddpm":
        return diffusion.p_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, use_graph=use_graph,
                                       model_kwargs={"y": y})
    return diffusion.ddim_sample_loop(m, shape, noise=xT, clip_denoised=False, noise_tape=tape, eta=eta, use_graph=use_graph,
                                      model_kwargs={"y": y})


def test_identities_and_kernel_count(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 3)
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    plain_jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    zero_jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=0.0, floor_weight=0.0, floor_height=0.3)
    foot_jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW, floor_height=FH)
    for use_graph in (True, False):
        for sampler, eta in (("ddpm", 0.0), ("ddim", 0.0)):
            a = _loop(diffusion, plain_jc, shape, xT, tape, _y(inp, **joint), sampler, eta, use_graph)
            b = _loop(diffusion, zero_jc, shape, xT, tape, _y(inp, **joint), sampler, eta, use_graph)
            assert torch.equal(a, b), (use_graph, sampler)
            c = _loop(diffusion, foot_jc, shape, xT, tape, _y(inp, **joint), sampler, eta, use_graph)
            assert not torch.equal(a, c)
    # a given mask equal to the derived one: the derivation reads each step's x0, so compare on one step's x0 through the hook
    x0 = torch.randn(B, 263, T, generator=torch.Generator().manual_seed(2)).cuda()
    lengths = inp["lengths"]
    kap = fo.derive_contact(x0.cpu(), mean, std, lengths).float()
    h1 = foot_guidance_hook(x0, mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, ITERS, CW, FW, FH, None, lengths)
    h2 = foot_guidance_hook(x0, mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, ITERS, CW, FW, FH, kap.cuda(), lengths)
    assert torch.equal(h1[0], h2[0]) and torch.equal(h1[1], h2[1])
    # ... and in a loop, with every step's x0 giving the same mask: a mask of zeros against a contact weight of 0
    only_floor = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=0.0, floor_weight=FW)
    zero_kappa = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW)
    a = _loop(diffusion, only_floor, shape, xT, tape, _y(inp, **joint))
    b = _loop(diffusion, zero_kappa, shape, xT, tape, _y(inp, foot_contact=torch.zeros(B, 4, T, dtype=torch.bool).cuda(), **joint))
    assert torch.equal(a, b)
    eng = cfg.model.engine()
    counts = {}
    for name, m in (("joint", plain_jc), ("foot", foot_jc)):
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        _loop(diffusion, m, shape, xT, tape, _y(inp, **joint))
        torch.cuda.synchronize()
        counts[name] = eng.launch_count()
    print("launches of a %d-step loop: joint %d, joint + foot %d" % (steps, counts["joint"], counts["foot"]))
    assert counts["joint"] == counts["foot"]


def _oracle_loop(sd, L, steps, inp, idx, control, foot_only, sampler="ddpm", eta=0.0, inpaint=None, arch="enc", den=None):
    mean, std, target, weight = control
    if foot_only:
        weight = torch.zeros_like(weight)
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    if den is None:
        make = deo.denoiser if arch == "dec" else po.enc_denoiser
        den = make(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    f = fo.guided_denoiser(den, mean, std, target[idx], weight[idx], STEP, ITERS, CW, FW, FH, None, inp["lengths"][idx])
    with torch.no_grad():
        return deo.sample_loop(f, tabs, [t[idx] for t in inp["tape"]], sampler=sampler, eta=eta, inpaint=inpaint)


def test_guided_loops_against_oracle_small(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    control = _control(B, T, 5)
    mean, std, target, weight = control
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW, floor_height=FH)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    g = torch.Generator().manual_seed(6)
    mask = torch.zeros(B, 263, 1, T, dtype=torch.bool)
    mask[..., : T // 4] = True
    motion = torch.randn(B, 263, 1, T, generator=g) * 0.5
    idx = list(range(B))
    for foot_only in (False, True):
        keys = {} if foot_only else joint
        for sampler, eta, inpaint in (("ddpm", 0.0, None), ("ddim", 0.0, None), ("ddim", 0.5, None), ("ddpm", 0.0, (mask, motion))):
            extra = dict(keys) if inpaint is None else dict(keys, inpainting_mask=mask.cuda(), inpainted_motion=motion.cuda())
            out = _loop(diffusion, jc, shape, xT, tape, _y(inp, **extra), sampler, eta)
            ref = _oracle_loop(sd, L, steps, inp, idx, control, foot_only, sampler, eta, inpaint)
            e = rel_err(out, ref)
            print("foot only %d, %s eta %.1f inpaint %d: engine vs oracle %.2e" % (foot_only, sampler, eta, inpaint is not None, e))
            assert e < RTOL
    prog = list(diffusion.p_sample_loop_progressive(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape,
                                                    model_kwargs={"y": _y(inp, **joint)}))
    loop = _loop(diffusion, jc, shape, xT, tape, _y(inp, **joint))
    assert torch.equal(prog[-1]["sample"], loop)
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    one = diffusion.p_sample(jc, prog[-2]["sample"], t, clip_denoised=False, model_kwargs={"y": _y(inp, **joint)}, noise=tape[-1])
    assert torch.equal(one["sample"], loop)
    dprog = list(diffusion.ddim_sample_loop_progressive(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape, eta=0.5,
                                                        model_kwargs={"y": _y(inp, **joint)}))
    assert torch.equal(dprog[-1]["sample"], _loop(diffusion, jc, shape, xT, tape, _y(inp, **joint), "ddim", 0.5))


def test_clip_decoder_against_oracle():
    B, T, steps, L = 3, 40, 6, 2
    cfg, diffusion, sd = _dec(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=12, scale=2.5, lengths=[40, 33, 20])
    control = _control(B, T, 9)
    mean, std, target, weight = control
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW, floor_height=FH)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    for foot_only, sampler, eta in ((False, "ddpm", 0.0), (True, "ddim", 0.5)):
        keys = {} if foot_only else dict(joint_target=target.cuda(), joint_weight=weight.cuda())
        out = _loop(diffusion, jc, (B, 263, 1, T), xT, tape, _y(inp, **keys), sampler, eta)
        ref = _oracle_loop(sd, L, steps, inp, list(range(B)), control, foot_only, sampler, eta, arch="dec")
        e = rel_err(out, ref)
        print("CLIP decoder, foot only %d, %s: engine vs oracle %.2e" % (foot_only, sampler, e))
        assert e < RTOL


def _contact_energy(sample, mean, std):
    """sum over (t, foot) of |p[t+1] - p[t]|^2 where the sample's own contact features say the foot is planted, the
    skating ratio (feet below 5 cm that move more than 2.5 cm horizontally) and the floor penetration (m, summed)"""
    xyz = ric_oracle.sample_to_xyz(sample.cpu(), mean, std).double()              # [B, J, 3, T]
    x = sample.cpu().double()[:, :, 0] * std.double()[None, :, None] + mean.double()[None, :, None]
    kap = (x[:, 259:263, :-1] > 0.5).double()                                      # [B, 4, T-1]
    feet = xyz[:, [7, 10, 8, 11]]                                                  # [B, 4, 3, T]
    d = feet[..., 1:] - feet[..., :-1]
    energy = float((kap * (d * d).sum(2)).sum())
    low = feet[:, :, 1, :-1] < 0.05
    slide = (d[:, :, [0, 2]] ** 2).sum(2).sqrt() > 0.025
    skate = float((low & slide).sum()) / max(1, int(low.sum()))
    pen = float((-xyz[:, :, 1]).clamp_min(0).sum())
    return energy, skate, pen


def test_headline_b64_against_oracle_and_effect():
    B, T, steps, L = 64, 196, 50, 8
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=2.5)
    control = _control(B, T, 7)
    mean, std, target, weight = control
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW, floor_height=FH)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    shape = (B, 263, 1, T)
    out = _loop(diffusion, jc, shape, xT, tape, _y(inp, joint_target=target.cuda(), joint_weight=weight.cuda()))
    plain = _loop(diffusion, cfg, shape, xT, tape, _y(inp))
    idx = [0, 31, 63]
    ref = _oracle_loop(sd, L, steps, inp, idx, control, False)
    e = rel_err(out[idx].cpu(), ref)
    eg, sg, pg = _contact_energy(out, mean, std)
    ep, sp, pp = _contact_energy(plain, mean, std)
    print("enc B=64 T=196 L=8 DDPM 50, K %d: engine vs oracle %.2e; contact energy guided %.4g, unguided %.4g (%.3f); "
          "skating %.3f vs %.3f; floor penetration %.4g vs %.4g m" % (ITERS, e, eg, ep, eg / ep, sg, sp, pg, pp))
    assert e < RTOL
    assert eg < ep


# ------------------------------------------------------------------------------------------------ state
def test_state_and_sharding(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 8)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS, contact_weight=CW, floor_weight=FW, floor_height=FH)
    plain_jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    shape = (B, 263, 1, T)
    _loop(diffusion, jc, shape, xT, tape, _y(inp, **joint))
    after = _loop(diffusion, cfg, shape, xT, tape, _y(inp))
    fresh, _, _ = _enc(L, steps)
    want = _loop(diffusion, fresh, shape, xT, tape, _y(inp))
    assert torch.equal(after, want)
    fresh.model.engine().close()
    # a plain joint-controlled loop after one with the foot terms equals it alone
    jwant = _loop(diffusion, plain_jc, shape, xT, tape, _y(inp, **joint))
    _loop(diffusion, jc, shape, xT, tape, _y(inp, **joint))
    assert torch.equal(_loop(diffusion, plain_jc, shape, xT, tape, _y(inp, **joint)), jwant)
    # Philox shards
    kw = {"y": _y(inp, **joint)}
    full = diffusion.p_sample_loop(jc, shape, clip_denoised=False, model_kwargs=kw, noise_seed=9)
    parts = []
    for lo, hi in ((0, 1), (1, 3)):
        parts.append(diffusion.p_sample_loop(jc, (hi - lo,) + shape[1:], clip_denoised=False, noise_seed=9, sample_index_base=lo,
                                             model_kwargs=parallel.shard_model_kwargs(kw, lo, hi)))
    assert torch.equal(torch.cat(parts), full)
    torch.cuda.synchronize()

