"""GPU: pseudo linear multistep sampling (plms_sample / plms_sample_loop / plms_sample_loop_progressive).

  * the PLMS epilogue bit for bit against a torch fp32 restatement of the reference's operations (Adams-Bashforth at
    cur_order 1-4, the pseudo improved-Euler step, including its i = -1 wrap), and three mutants of that restatement
    that it must tell apart;
  * every case of tests/golden/plms_small.npz (the reference's own output) within 1e-3 relative error, except the two
    coarse-schedule cases held to COARSE_TOL (see below);
  * plms_sample with an empty history (old_out = {'old_eps': []}) at orders 1 and 2: one Adams-Bashforth forward;
  * BASELINE config 2's shape (B=64, T=196, CFG 2.5, L=8, 50 steps) at orders 2 and 4 against the fp32 oracle on 3 samples;
  * graph replay == plain launches == chained plms_sample == the progressive form, bit for bit; one generator draw;
    the Philox x_T split-invariant; an Adams-Bashforth step launches what a DDIM step launches."""
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm.parallel import shard_model_kwargs
from conftest import default_args, rel_err
from oracle import gen_golden_plms as gp
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
# The 6-step fixture at orders 3 and 4 (and every intermediate sample of order 4) measured 1.2e-3 to 3.7e-3 against the
# reference, while its epilogue is bit-exact against a restatement fed with the engine's own forwards (the first two
# tests).  Near the noisy end of a 6-step cosine schedule sqrt(1/abar - 1) reaches ~1e2, so pred' = sr*x - srm1*eps'
# scales the forwards' fp16 rounding up, and the Adams-Bashforth weights add to it; guidance 7.5 on one sample adds
# more.  Those cases are held to this bound; every other case, and the 50-step c2 shape at orders 2 and 4, to RTOL.
COARSE_TOL = 5e-3


def _enc(layers, steps, seed):
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=layers, diffusion_steps=steps),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=layers, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion, sd


def _y(inp, scale=True):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda())
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _small():
    c = gp.ENC
    cfg, model, diffusion, _ = _enc(c["L"], c["steps"], c["weights_seed"])
    inp, shape, imask, motion = gp.enc_inputs()
    return cfg, model, diffusion, inp, shape, imask, motion


# ---------------------------------------------------------------------------------------------------------------------
def _rows(diffusion, i):
    r = torch.from_numpy(diffusion.schedule_rows(0.0))[i]
    return r[3], r[4], r[5], r[6]                       # sr, srm1, sqrt(abp), sqrt(1 - abp): fp32, as the reference


def _sample(diffusion, x, i, ep, x0, sq_row=None):
    """pred' -> mean -> (t != 0) blend (gaussian_diffusion.py:1065-1072), torch fp32 on the CPU."""
    sr, srm1, sq, s1 = _rows(diffusion, i)
    if sq_row is not None:
        sq = _rows(diffusion, sq_row)[2]
    mean = (sr * x - srm1 * ep) * sq + s1 * ep
    nz = torch.tensor(0.0 if i == 0 else 1.0)
    return mean * nz + x0 * (1 - nz)


def _eps(diffusion, x, i, x0):
    sr, srm1, _, _ = _rows(diffusion, i)
    return (sr * x - x0) / srm1


def test_epilogue_adams_bashforth_bit_exact():
    cfg, _, diffusion, inp, shape, _, _ = _small()
    y = _y(inp)
    x = inp["tape"][0].cuda()
    gen = torch.Generator().manual_seed(3)
    hist = [torch.randn(shape, generator=gen) for _ in range(5)]
    i = 3
    t = torch.full((shape[0],), i, dtype=torch.long, device="cuda")
    # n_old == 0: old_out = {'old_eps': []}, which the reference runs as one Adams-Bashforth forward at cur_order 1
    for order, n_old in ((1, 0), (2, 0), (1, 1), (2, 1), (3, 2), (4, 3), (4, 5), (2, 4)):
        old = [h.cuda() for h in hist[:n_old]]
        out = diffusion.plms_sample(cfg, x, t, clip_denoised=False, model_kwargs={"y": y}, order=order,
                                    old_out={"old_eps": list(old)})
        x0, xc = out["pred_xstart"].cpu(), x.cpu()
        eps = _eps(diffusion, xc, i, x0)
        if out["old_eps"]:                              # (order 1 pops this step's own eps again)
            assert torch.equal(out["old_eps"][-1].cpu(), eps), (order, n_old)
        cpu_hist = [h.clone() for h in hist[:n_old]] + [eps]
        ep = po.ab_combine(cpu_hist, order)
        got = out["sample"].cpu()
        assert torch.equal(got, _sample(diffusion, xc, i, ep, x0)), (order, n_old)
        assert len(out["old_eps"]) == (n_old if n_old + 1 >= order else n_old + 1)      # :1068-1069
        cur = min(order, n_old + 1)
        if cur == 3:                                    # mutant: multiply by 1/12 instead of dividing by 12
            e = cpu_hist
            bad = (23 * e[-1] - 16 * e[-2] + 5 * e[-3]) * (1.0 / 12)
            assert not torch.equal(got, _sample(diffusion, xc, i, bad, x0))
        if cur >= 2 and n_old >= 2:                     # mutant: history slots reversed
            bad = po.ab_combine(cpu_hist[:-1][::-1] + [eps], order)
            assert not torch.equal(got, _sample(diffusion, xc, i, bad, x0))
        assert not torch.equal(got, _sample(diffusion, xc, i, ep, x0, sq_row=i - 1))   # mutant: sqrt(abp) of row i-1


@pytest.mark.parametrize("i", [3, 0])
def test_epilogue_improved_euler_bit_exact(i):
    """The second forward runs at schedule index i - 1; at i = 0 that is the last index (the reference indexes -1)."""
    cfg, _, diffusion, inp, shape, _, _ = _small()
    y = _y(inp)
    x = inp["tape"][0].cuda()
    t = torch.full((shape[0],), i, dtype=torch.long, device="cuda")
    for clip in (False, True):
        out = diffusion.plms_sample(cfg, x, t, clip_denoised=clip, model_kwargs={"y": y}, order=2)
        x0, xc = out["pred_xstart"].cpu(), x.cpu()
        eps0 = _eps(diffusion, xc, i, x0)
        assert len(out["old_eps"]) == 1 and torch.equal(out["old_eps"][0].cpu(), eps0)
        _, _, sq, s1 = _rows(diffusion, i)
        mean1 = x0 * sq + s1 * eps0
        j = i - 1 if i > 0 else diffusion.num_timesteps - 1
        x0b = cfg(mean1.cuda(), torch.full((shape[0],), diffusion.timestep_map[j], dtype=torch.long, device="cuda"),
                  y=y).cpu()
        if clip:
            x0b = x0b.clamp(-1, 1)
        eps2 = _eps(diffusion, mean1, j, x0b)
        ep = (eps0 + eps2) / 2
        got = out["sample"].cpu()
        assert torch.equal(got, _sample(diffusion, xc, i, ep, x0)), clip
        if i > 0:
            assert not torch.equal(got, _sample(diffusion, xc, i, ep, x0, sq_row=i - 1))


# ---------------------------------------------------------------------------------------------------------------------
def test_golden_cases(golden):
    g = golden("plms_small.npz")
    cfg, model, diffusion, inp, shape, imask, motion = _small()
    xT = inp["tape"][0].cuda()

    def loop(m, order, scale=True, **kw):
        y = _y(inp, scale)
        y.update(kw.pop("extra", {}))
        clip = kw.pop("clip", False)
        outs = [diffusion.plms_sample_loop(m, shape, noise=xT, clip_denoised=clip, model_kwargs={"y": y}, order=order,
                                           use_graph=ug, **kw) for ug in (True, False)]
        assert torch.equal(outs[0], outs[1]), (order, kw)
        return outs[0]
    assert rel_err(loop(cfg, 2), g["enc_o2"]) < RTOL
    assert rel_err(loop(cfg, 3), g["enc_o3"]) < COARSE_TOL
    steps = [o["sample"] for o in diffusion.plms_sample_loop_progressive(cfg, shape, noise=xT, clip_denoised=False,
                                                                         model_kwargs={"y": _y(inp)}, order=4)]
    assert len(steps) == len(g["enc_o4_steps"])
    errs = [rel_err(s, g["enc_o4_steps"][k]) for k, s in enumerate(steps)]
    print("PLMS order 4, per-step relative error vs the reference:", " ".join("%.2e" % e for e in errs))
    assert max(errs) < COARSE_TOL, errs
    assert torch.equal(loop(cfg, 4), steps[-1])
    assert rel_err(loop(cfg, 2, clip=True), g["enc_o2_clip"]) < RTOL
    assert rel_err(loop(cfg, 2, extra=dict(inpainting_mask=imask.cuda(), inpainted_motion=motion.cuda())),
                   g["enc_o2_inpaint"]) < RTOL
    assert rel_err(loop(cfg, 2, skip_timesteps=5), g["enc_o2_skip5"]) < RTOL
    assert rel_err(loop(model, 2, scale=False), g["enc_o2_noguide"]) < RTOL


def test_dip_golden(golden):
    c = gp.DIP
    args = default_args(layers=c["L"], diffusion_steps=c["steps"], arch="trans_dec", text_encoder_type="bert",
                        context_len=c["ctx"], pred_len=c["pred"])
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                                   seed=c["weights_seed"]))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp, enc, tmask, prefix = gp.dip_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             scale=inp["scale"].cuda(), prefix=prefix.cuda())
    shape = (c["B"], 263, 1, c["pred"])
    outs = [diffusion.plms_sample_loop(cfg, shape, noise=inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": y},
                                       order=2, use_graph=ug) for ug in (True, False)]
    assert torch.equal(outs[0], outs[1])
    assert rel_err(outs[0], golden("plms_small.npz")["dip_o2"]) < RTOL


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [2, 4])
def test_c2_shape_50_steps_vs_oracle(order):
    B, T, steps = 64, 196, 50
    cfg, _, diffusion, sd = _enc(8, steps, 0)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    out = diffusion.plms_sample_loop(cfg, (B, 263, 1, T), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                     model_kwargs={"y": _y(inp)}, order=order)
    assert torch.isfinite(out).all()
    idx = [0, 31, 63]
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = po.enc_denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    ref = po.plms_loop(f, tabs, inp["tape"][0][idx], order)
    err = rel_err(out[idx], ref)
    print("PLMS order %d, B=64 x 50 steps x CFG 2.5: Frobenius-relative %.3e" % (order, err))
    assert err < RTOL


def test_loop_forms_generator_and_launches():
    cfg, _, diffusion, inp, shape, _, _ = _small()
    y = _y(inp)
    xT = inp["tape"][0].cuda()
    n = diffusion.num_timesteps
    loop = diffusion.plms_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y}, order=3)
    x, old = xT, None
    for i in range(n)[::-1]:
        o = diffusion.plms_sample(cfg, x, torch.full((shape[0],), i, dtype=torch.long, device="cuda"),
                                  clip_denoised=False, model_kwargs={"y": y}, order=3, old_out=old)
        x, old = o["sample"], o
    assert torch.equal(x, loop)
    assert torch.equal(xT, inp["tape"][0].cuda())            # the caller's x_T is not clobbered by the in-place loop
    # one generator draw: x_T
    torch.cuda.manual_seed(123)
    diffusion.plms_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": y}, order=2)
    after = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(123)
    torch.randn(shape, device="cuda")
    assert torch.equal(after, torch.cuda.get_rng_state())
    # an Adams-Bashforth step launches what a DDIM step launches (continuation calls: no first step, no copies)
    eng = cfg.model.engine()
    diffusion.plms_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y}, order=2)
    for use_graph in (True, False):
        eng.plms_loop_range(2, n - 1, 1, xT, None, 0, use_graph)
        eng.launch_count(reset=True)
        eng.plms_loop_range(2, n - 2, n - 1, None, None, 0, use_graph)
        plms = eng.launch_count(reset=True)
        tape = torch.zeros((n - 1,) + tuple(shape), device="cuda")
        eng.sample_loop_range(b200mdm._lib.MODE_DDIM, n - 2, n - 1, xT, None, tape, 0, use_graph)
        ddim = eng.launch_count(reset=True)
        assert plms == ddim, (use_graph, plms, ddim)
        torch.cuda.synchronize()


def test_philox_x_T_is_split_invariant():
    cfg, _, diffusion, _ = _enc(2, 6, 1)
    B, T = 64, 24
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=4)
    shape = (B, 263, 1, T)
    full = diffusion.plms_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": _y(inp)}, noise_seed=77)
    halves = []
    for lo in (0, 32):
        part = shard_model_kwargs({"y": _y(inp)}, lo, lo + 32)
        halves.append(diffusion.plms_sample_loop(cfg, (32, 263, 1, T), clip_denoised=False, model_kwargs=part,
                                                 noise_seed=77, sample_index_base=lo))
    assert torch.equal(full, torch.cat(halves))
