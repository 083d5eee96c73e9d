"""GPU: joint-position control (JointControlSampleModel; joint_guidance_step_kernel, DESIGN.md "Joint-position control").

  1. the guidance iterations alone (b200mdm_test_joint_guidance) against the fp64 oracle within the bound of DESIGN.md,
     for root / sparse keyframe / all-joint weights, K = 1 and 10, T = 1, 2, 60, 196, 255, HumanML3D and KIT; four
     mutants (sign flip, yaw adjoint dropped, velocity adjoint off by one frame, std left out) miss that bound 8-fold;
  2. guidance with all-zero weights gives the unguided DDPM / DDIM loops bit for bit (graph and eager, with inpainting,
     soft weights and clip_denoised); a guided step launches exactly one kernel more than an unguided one;
  3. guided loops against the fp32 oracle (oracle/joint_control_oracle.guided_denoiser) within 1e-3: DDPM, DDIM eta 0
     and 0.5, CFG 2.5, with inpainting, at a small shape; B = 64, T = 196, L = 8, 50 DDPM steps for the encoder and the
     CLIP decoder, the oracle following three samples;
  4. the loss never increases over the iterations at the tested step, and the final samples' weighted joint error
     (through sample_to_xyz) is below 0.95 of the unguided samples' at the headline shape;
  5. set_cond clears the guidance; a Philox loop split into batch halves equals the batch bit for bit; the C ABI's
     ENOTIMPL refusals."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from b200mdm.engine import joint_guidance_hook
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ric_oracle
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
U32 = 2.0 ** -24
EPS_G = 2.0 ** -12          # relative error of the kernel's guidance displacement (DESIGN.md)
EPS_L = 2.0 ** -16          # relative error of its per-iteration loss


def _positions(x, mean, std):
    """recover_from_ric of normalised x [B, D, T] -> [B, J, 3, T] (fp64)"""
    D = x.shape[1]
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    return ric_oracle.recover_from_ric(data, jo.n_joints(D)).permute(0, 2, 3, 1)


def _weights(kind, B, J, T, g):
    w = torch.zeros(B, J, T, dtype=torch.float64)
    if kind == "root":
        w[:, 0] = 1.0
    elif kind == "sparse":                                           # wrists and feet at a few keyframes
        for j in (20, 21, 10, 11) if J == 22 else (7, 4, 19, 20):
            frames = torch.randint(0, T, (max(1, T // 20),), generator=g)
            w[:, j, frames] = 0.5 + torch.rand(len(frames), generator=g, dtype=torch.float64)
    else:
        w[:] = 0.2 + torch.rand(B, J, T, generator=g, dtype=torch.float64)
    return w


def _hook_case(D, T, kind, seed):
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    B = 3
    x0 = (torch.randn(B, D, T, generator=g) * 0.7).float()
    target = _positions(torch.randn(B, D, T, generator=g) * 0.7, mean, std) + 0.3 * torch.randn(B, J, 3, T, generator=g, dtype=torch.float64)
    weight = _weights(kind, B, J, T, g)
    p0 = _positions(x0, mean, std)
    xz = torch.cat([p0[:, :, [0, 2]].reshape(B, -1), target[:, :, [0, 2]].reshape(B, -1)], 1)
    extent = float(xz.max() - xz.min()) + 1.0
    step = jo.step_bound(std, weight, extent, T)
    return x0, mean, std, target.float(), weight.float(), step


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [1, 2, 60, 196, 255])
def test_hook_against_fp64_oracle_and_mutants(D, T):
    for kind in ("root", "sparse", "all"):
        for K in (1, 10):
            x0, mean, std, target, weight, step = _hook_case(D, T, kind, seed=D * 1000 + T + K)
            got, loss = joint_guidance_hook(x0.cuda(), mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), step, K)
            got, loss = got.double().cpu(), loss.double().cpu()
            want, want_loss = jo.guide(x0, mean, std, target, weight, step, K)
            R = jo.ric_features(jo.n_joints(D))
            assert torch.equal(got[:, R:], x0[:, R:].double())        # every other feature bit for bit
            disp = float((want - x0.double()).abs().max())
            bound = EPS_G * disp + 2 * U32 * K * float(x0.abs().max())
            err = float((got - want).abs().max())
            lerr = float(((loss - want_loss).abs() / (EPS_L * want_loss[0].clamp_min(1e-30))).max())
            print("D %d T %3d %-6s K %2d: |dx| %.2e, err / bound %.3f, loss err / bound %.3f, loss %.4g -> %.4g"
                  % (D, T, kind, K, disp, err / bound, lerr, float(want_loss[0].sum()), float(want_loss[-1].sum())))
            assert err <= bound and lerr <= 1.0, (kind, K)
            assert bool((loss[1:] <= loss[:-1] * (1 + 1e-6)).all()), (kind, K)   # the loss does not increase
            if T >= 60:
                for m in ("sign", "no_yaw", "vel_shift", "no_std"):
                    mut, _ = jo.guide_manual(x0, mean, std, target, weight, step, K, mutant=m)
                    miss = float((got - mut.double()).abs().max()) / bound
                    assert miss >= 8.0, (kind, K, m, miss)


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


def _control(B, T, seed, keyframes=True):
    """targets [B, 22, 3, T] (the positions of a random normalised motion) and weights: the pelvis on every frame, the
    wrists at a few keyframes"""
    g = torch.Generator().manual_seed(seed)
    mean, std = jo.motion_stats(263)
    target = _positions(torch.randn(B, 263, T, generator=g) * 0.5, mean, std).float()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    if keyframes:
        for j in (20, 21):
            weight[:, j, torch.arange(T // 4, T, max(1, T // 4))] = 1.0
    return mean, std, target, weight


def _y(inp, **extra):
    return dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
                scale=inp["scale"].cuda(), **extra)


STEP, ITERS = 2e-4, 10


@pytest.fixture(scope="module")
def small():
    B, T, steps, L = 3, 40, 6, 2
    cfg, diffusion, sd = _enc(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=11, scale=2.5)
    return B, T, steps, L, cfg, diffusion, sd, inp


def test_zero_weights_are_the_unguided_loop(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 3)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    g = torch.Generator().manual_seed(4)
    mask = torch.rand(B, 263, 1, T, generator=g) < 0.3
    soft = torch.rand(B, 263, 1, T, generator=g)
    motion = torch.randn(B, 263, 1, T, generator=g)
    zero = dict(joint_target=target.cuda(), joint_weight=torch.zeros_like(weight).cuda())
    variants = [dict(), dict(inpainting_mask=mask.cuda(), inpainted_motion=motion.cuda()),
                dict(inpainting_weight=soft.cuda(), inpainted_motion=motion.cuda())]
    for extra in variants:
        for clip in (False, True):
            for use_graph in (True, False):
                for fn, kw in ((diffusion.p_sample_loop, {}), (diffusion.ddim_sample_loop, {"eta": 0.0})):
                    plain = fn(cfg, (B, 263, 1, T), noise=xT, clip_denoised=clip, noise_tape=tape, use_graph=use_graph,
                               model_kwargs={"y": _y(inp, **extra)}, **kw)
                    guided = fn(jc, (B, 263, 1, T), noise=xT, clip_denoised=clip, noise_tape=tape, use_graph=use_graph,
                                model_kwargs={"y": _y(inp, **extra, **zero)}, **kw)
                    assert torch.equal(plain, guided), (sorted(extra), clip, use_graph, fn.__name__)
    eng = cfg.model.engine()
    counts = {}
    for name, m, y in (("plain", cfg, _y(inp)), ("guided", jc, _y(inp, **zero))):
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        diffusion.p_sample_loop(m, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": y})
        torch.cuda.synchronize()
        counts[name] = eng.launch_count()
    print("launches of a %d-step loop: unguided %d, guided %d" % (steps, counts["plain"], counts["guided"]))
    assert counts["guided"] - counts["plain"] == steps


def _oracle_loop(sd, L, steps, inp, idx, control, sampler="ddpm", eta=0.0, inpaint=None, dec=False):
    mean, std, target, weight = control
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    if dec:
        den = deo.denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    else:
        den = po.enc_denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    f = jo.guided_denoiser(den, mean, std, target[idx], weight[idx], STEP, ITERS)
    with torch.no_grad():
        return deo.sample_loop(f, tabs, [t[idx] for t in inp["tape"]], sampler=sampler, eta=eta, inpaint=inpaint)


def test_guided_loops_against_oracle_small(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    control = _control(B, T, 5)
    mean, std, target, weight = control
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    g = torch.Generator().manual_seed(6)
    mask = torch.zeros(B, 263, 1, T, dtype=torch.bool)
    mask[..., : T // 4] = True
    motion = torch.randn(B, 263, 1, T, generator=g) * 0.5
    idx = list(range(B))
    cases = [("ddpm", 0.0, None), ("ddim", 0.0, None), ("ddim", 0.5, None), ("ddpm", 0.0, (mask, motion))]
    for sampler, eta, inpaint in cases:
        extra = dict(joint) if inpaint is None else dict(joint, inpainting_mask=mask.cuda(), inpainted_motion=motion.cuda())
        if sampler == "ddpm":
            out = diffusion.p_sample_loop(jc, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape,
                                          model_kwargs={"y": _y(inp, **extra)})
        else:
            out = diffusion.ddim_sample_loop(jc, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape, eta=eta,
                                             model_kwargs={"y": _y(inp, **extra)})
        ref = _oracle_loop(sd, L, steps, inp, idx, control, sampler, eta, inpaint)
        e = rel_err(out, ref)
        print("guided %s eta %.1f inpaint %s: engine vs oracle %.2e" % (sampler, eta, inpaint is not None, e))
        assert e < RTOL
    # the single-step and progressive forms are the loop's steps
    prog = list(diffusion.p_sample_loop_progressive(jc, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape,
                                                    model_kwargs={"y": _y(inp, **joint)}))
    loop = diffusion.p_sample_loop(jc, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape,
                                   model_kwargs={"y": _y(inp, **joint)})
    assert torch.equal(prog[-1]["sample"], loop)
    t = torch.zeros(B, dtype=torch.long, device="cuda")
    one = diffusion.p_sample(jc, prog[-2]["sample"], t, clip_denoised=False, model_kwargs={"y": _y(inp, **joint)},
                             noise=tape[-1])
    assert torch.equal(one["sample"], loop) and torch.equal(one["pred_xstart"], loop)   # i = 0: the sample is x0
    ddim = diffusion.ddim_sample(jc, prog[-2]["sample"], t, clip_denoised=False, model_kwargs={"y": _y(inp, **joint)},
                                 noise=tape[-1])
    assert torch.isfinite(ddim["sample"]).all()


def _weighted_error(sample, mean, std, target, weight):
    xyz = ric_oracle.sample_to_xyz(sample.cpu(), mean, std).double()               # [B, J, 3, T]
    d = (xyz - target.double()) ** 2
    return float((weight.double()[:, :, None] * d).sum()) ** 0.5


@pytest.mark.parametrize("arch", ["enc", "dec"])
def test_headline_b64_against_oracle_and_control_takes_effect(arch):
    B, T, steps, L = 64, 196, 50, 8
    cfg, diffusion, sd = _enc(L, steps) if arch == "enc" else _dec(L, steps)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=2.5)
    control = _control(B, T, 7)
    mean, std, target, weight = control
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    y = _y(inp, joint_target=target.cuda(), joint_weight=weight.cuda())
    out = diffusion.p_sample_loop(jc, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": y})
    plain = diffusion.p_sample_loop(cfg, (B, 263, 1, T), noise=xT, clip_denoised=False, noise_tape=tape,
                                    model_kwargs={"y": _y(inp)})
    idx = [0, 31, 63]
    ref = _oracle_loop(sd, L, steps, inp, idx, control, dec=arch == "dec")
    e = rel_err(out[idx].cpu(), ref)
    eg, ep = _weighted_error(out, mean, std, target, weight), _weighted_error(plain, mean, std, target, weight)
    print("%s B=64 T=196 L=8 DDPM 50, K %d: engine vs oracle %.2e; weighted joint error guided %.4g, unguided %.4g (%.3f)"
          % (arch, ITERS, e, eg, ep, eg / ep))
    assert e < RTOL
    # the synthetic weights do not carry the earlier steps' guidance into their x0 predictions, so only the last step's
    # K iterations act on the final sample (measured: 0.897 of the unguided error for the encoder, 0.889 for the decoder)
    assert eg < 0.95 * ep


# ------------------------------------------------------------------------------------------------ state
def test_state_sharding_and_refusals(small):
    B, T, steps, L, cfg, diffusion, sd, inp = small
    mean, std, target, weight = _control(B, T, 8)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    shape = (B, 263, 1, T)
    guided = diffusion.p_sample_loop(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": _y(inp, **joint)})
    after = diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": _y(inp)})
    fresh, _, _ = _enc(L, steps)
    want = diffusion.p_sample_loop(fresh, shape, noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": _y(inp)})
    assert torch.equal(after, want) and not torch.equal(guided, want)
    fresh.model.engine().close()
    # Philox shards
    kw = {"y": _y(inp, **joint)}
    full = diffusion.p_sample_loop(jc, shape, clip_denoised=False, model_kwargs=kw, noise_seed=9)
    parts = []
    for lo, hi in ((0, 1), (1, 3)):
        parts.append(diffusion.p_sample_loop(jc, (hi - lo,) + shape[1:], clip_denoised=False, noise_seed=9, sample_index_base=lo,
                                             model_kwargs=parallel.shard_model_kwargs(kw, lo, hi)))
    assert torch.equal(torch.cat(parts), full)
    # C ABI refusals while the guidance is set
    eng = cfg.model.engine()
    lib = eng.lib
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())                                        # noqa: E731
    x = xT.contiguous()
    out = torch.empty_like(x)

    def arm():
        eng.set_cond(B, T, _y(inp), True, torch.device("cuda"))
        eng.set_schedule(diffusion.schedule_rows(0.0), diffusion._timestep_map(), key=None)
        eng.set_schedule_next(diffusion.schedule_next_rows())
        eng.set_schedule_dpm(diffusion.schedule_dpm_rows())
        eng.set_schedule_vb(diffusion.schedule_vb_rows())
        eng.set_joint_guidance(mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, ITERS)
    arm()
    calls = {
        "plms": lambda: lib.b200mdm_plms_loop_range(eng.h, 2, steps - 1, steps, p(x), p(out), 0, 1, s),
        "dpm": lambda: lib.b200mdm_dpm_loop_range(eng.h, 2, steps - 1, steps, p(x), p(out), 0, 1, s),
        "reverse": lambda: lib.b200mdm_ddim_reverse_loop_range(eng.h, 0, steps, p(x), p(out), 0, 1, s),
        "reverse_step": lambda: lib.b200mdm_sample_step(eng.h, _lib.MODE_DDIM_REVERSE, 0, p(x), None, 0, p(out), None, s),
        "vb": lambda: lib.b200mdm_vb_loop_range(eng.h, steps - 1, steps, p(x), None, 0, _lib.FLAG_PHILOX_NOISE, None, None, 1, s),
    }
    for name, call in calls.items():
        assert call() == _lib.ENOTIMPL, name
        assert b"joint-position control" in lib.b200mdm_last_error(), name
    ln = (ctypes.c_int64 * B)(*([T] * B))
    assert lib.b200mdm_set_handshake(eng.h, 4, ln, None, s) == _lib.ENOTIMPL
    eng.set_cond(B, T, _y(inp), True, torch.device("cuda"))
    eng.set_handshake(4, B, T, {})
    assert lib.b200mdm_set_joint_guidance(eng.h, p(mean.cuda()), p(std.cuda()), p(target.cuda()), p(weight.cuda()),
                                          ctypes.c_float(STEP), ITERS, s) == _lib.ENOTIMPL
    args = default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    dip, _ = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(dip, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=1, cond_dim=768, seed=2))
    dip.to("cuda").eval()
    deng = dip.engine()
    assert deng.lib.b200mdm_set_joint_guidance(deng.h, p(mean.cuda()), p(std.cuda()), p(target.cuda()), p(weight.cuda()),
                                               ctypes.c_float(STEP), ITERS, s) == _lib.ENOTIMPL
    torch.cuda.synchronize()
