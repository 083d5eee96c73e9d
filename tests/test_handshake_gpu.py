"""GPU: long motions from chained windows (HandshakeSampleModel; the handshake inside blend_split_kernel).

  * the blend kernel alone (b200mdm_test_blend_handshake) against fp64 within a per-element bound derived from its
    arithmetic; four mutants of the restatement (alpha reversed, suffix frame off by one, a partner across a
    motion_start, the guidance scale of the wrong window) miss that bound at least 8-fold;
  * every entry of tests/golden/handshake_small.npz (the unmodified reference's samplers around the oracle's wrapper)
    and of the full-depth handshake_c1.npz within 1e-3 relative; DPM-Solver++ orders 1 and 2 against
    oracle/dpm_oracle.py with the wrapper;
  * the two copies of every handshake frame are bit-identical in the final samples of DDPM, DDIM and DPM-Solver++
    (the last step's sample is a function of the blended x0 alone); PLMS is reported;
  * h = 0 and an all-True motion_start give the plain model's loop bit for bit;
  * one engine across handshake / plain / other-layout loops and a bare forward equals a fresh engine bit for bit;
  * a Philox loop split into two motion-aligned shards equals the whole batch bit for bit;
  * the headline shape (64 windows as 8 motions of 8, h = 20, 50 DDIM steps, CFG 2.5) against the fp32 oracle following
    one whole motion."""
import ctypes
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import default_args, rel_err
from oracle import dpm_oracle as do
from oracle import handshake_oracle as ho
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
# PLMS on the 4-step fixture measured 1.05e-3 against the reference (the other samplers 6.3e-4 to 7.0e-4 on the same
# windows).  Near the noisy end of a 4-step cosine schedule sqrt(1/abar - 1) is large, so PLMS's pred' = sr*x - srm1*eps'
# scales the forwards' fp16 rounding up and the Adams-Bashforth weights add to it: the effect tests/test_plms_gpu.py
# documents for short schedules.  The handshake itself is a convex blend and adds no amplification.
PLMS_TOL = 2e-3
gh = importlib.import_module("oracle.gen_golden_handshake")
deo = importlib.import_module("oracle.dec_emb_oracle")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _model(layers, steps, seed, guided=True, **over):
    args = default_args(layers=layers, diffusion_steps=steps, **over)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    kw = dict(arch="trans_dec", cond_dim=512) if over.get("arch") == "trans_dec" else {}
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=layers, seed=seed, **kw))
    model.to("cuda").eval()
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), diffusion


def _y(inp, y, scale=True, **extra):
    out = dict(mask=y["mask"].cuda(), lengths=y["lengths"].cuda(), text_embed=y["text_embed"].cuda(),
               motion_start=y["motion_start"].cuda(), **extra)
    if scale:
        out["scale"] = inp["scale"].cuda()
    return out


def _pairs(y, h, T):
    return ho.pairs(len(y["lengths"]), T, h, y["lengths"].cpu(), y["motion_start"].cpu())


def _dup_equal(sample, y, h, T):
    """Every handshake frame's two copies are bit-identical."""
    return all(torch.equal(sample[p, ..., n_p - h + j], sample[b, ..., j]) for p, b, n_p in _pairs(y, h, T) for j in range(h))


# ------------------------------------------------------------------------------------------------ the kernel alone
def _ref64(hres, scale, B, T, d, s_off, h, lengths, starts, halves, wrong_scale=False, **mutant):
    """fp64 g of the frame rows: CFG blend of hi + lo, then the handshake (oracle/handshake_oracle.blend)."""
    S = T + s_off
    v = hres.double()
    val = v[:, :d] + v[:, d:]
    c = val[: B * S].view(B, S, d)[:, s_off:]
    if halves == 1:
        D = c
    else:
        u = val[B * S:].view(B, S, d)[:, s_off:]
        sc = scale.double().view(B, 1, 1)
        D = u + sc * (c - u)
    D = D.permute(0, 2, 1)                                                        # [B, d, T]
    out = ho.blend(D, h, lengths, starts, **mutant)
    if wrong_scale:                                                               # the partner blended with b's scale
        out = D.clone()
        for p, b, n_p in ho.pairs(B, T, h, lengths, starts):
            for j in range(h):
                a = (j + 1) / (h + 1)
                fp = n_p - h + j
                up, cp = u[p, fp], c[p, fp]
                wrong = up + scale[b].double() * (cp - up)
                out[p, :, fp] = out[b, :, j] = (1 - a) * wrong + a * D[b, :, j]
    return out.permute(0, 2, 1).reshape(B * T, d), D.permute(0, 2, 1).reshape(B * T, d)


def _bound(hres, scale, B, T, d, s_off, h, lengths, starts, halves, want, D):
    """Per-element bound on the kernel's fp32 arithmetic.  A row's operand: hi + lo in fp32 (u|h|), then the CFG blend
    (u|c - u|, u|s (c - u)|, u|v|): 4u * mag with mag = |u| + |s||c - u| + |v| (|v| without guidance).  A handshake
    row: both operands' errors carried by weights <= 1, and the roundings of a, 1 - a, the two products and the sum,
    each within u(|v_a| + |v_b|): 8u (mag_a + mag_b).  Then the [hi | lo] split of the result: 2^-22 |g| relative, and
    2^-25 absolute where lo falls into fp16's subnormal range."""
    u32 = 2.0 ** -24
    S = T + s_off
    val = hres.double()[:, :d] + hres.double()[:, d:]
    if halves == 2:
        cc = val[: B * S].view(B, S, d)[:, s_off:].reshape(B * T, d)
        uu = val[B * S:].view(B, S, d)[:, s_off:].reshape(B * T, d)
        sc = scale.double().repeat_interleave(T).view(-1, 1)
        mag = uu.abs() + sc.abs() * (cc - uu).abs() + D.abs()
    else:
        mag = D.abs()
    hs_mag = torch.zeros_like(mag)
    for p, b, n_p in ho.pairs(B, T, h, lengths, starts):
        for j in range(h):
            rp, rb = p * T + n_p - h + j, b * T + j
            hs_mag[rp] = hs_mag[rb] = mag[rp] + mag[rb]
    return 4 * u32 * mag + 8 * u32 * hs_mag + 2.0 ** -22 * want.abs() + 2.0 ** -25


@pytest.mark.parametrize("halves", [1, 2])
def test_blend_kernel_vs_fp64_and_mutants(halves):
    lib = _lib.load()
    B, T, d, s_off, h = 5, 24, 512, 1, 6
    lengths, starts = [24, 20, 24, 16, 24], [1, 0, 0, 1, 0]
    S = T + s_off
    g = torch.Generator(device="cuda").manual_seed(23 + halves)
    x = torch.randn(halves * B * S, d, device="cuda", generator=g) * 1.5
    hi = x.half()
    hres = torch.cat([hi, (x - hi.float()).half()], 1).contiguous()
    scale = torch.tensor([2.5, 1.0, 7.5, 0.0, 4.0], device="cuda") if halves == 2 else None
    g16 = torch.empty(B * T, 3 * d, device="cuda", dtype=torch.float16)
    ln = np.array(lengths, dtype=np.int64)
    ms = np.array(starts, dtype=np.uint8)
    _lib.check(lib.b200mdm_test_blend_handshake(_p(hres), _p(scale), _p(g16), B, T, d, s_off, halves, h,
                                                ln.ctypes.data_as(ctypes.c_void_p), ms.ctypes.data_as(ctypes.c_void_p),
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    got = (g16[:, :d].double() + g16[:, d:2 * d].double()).cpu()
    assert torch.equal(g16[:, :d], g16[:, 2 * d:])
    hres_c, sc_c = hres.cpu(), scale.cpu() if scale is not None else None
    lt, mt = torch.tensor(lengths), torch.tensor(starts, dtype=torch.bool)
    want, D = _ref64(hres_c, sc_c, B, T, d, s_off, h, lt, mt, halves)
    bound = _bound(hres_c, sc_c, B, T, d, s_off, h, lt, mt, halves, want, D)
    ratio = float(((got - want).abs() / bound).max())
    print("halves %d: max |err| / bound = %.3f" % (halves, ratio))
    assert ratio <= 1.0
    # the copies agree bit for bit
    for p, b, n_p in ho.pairs(B, T, h, lt, mt):
        assert torch.equal(g16[p * T + n_p - h: p * T + n_p], g16[b * T: b * T + h])
    mutants = [dict(alpha_reversed=True), dict(suffix_shift=-1), dict(ignore_motion_start=True)]
    if halves == 2:
        mutants.append(dict(wrong_scale=True))
    for mut in mutants:
        wm, _ = _ref64(hres_c, sc_c, B, T, d, s_off, h, lt, mt, halves, **mut)
        miss = float(((got - wm).abs() / bound).max())
        print("mutant %s misses the bound %.3g-fold" % (mut, miss))
        assert miss >= 8.0, mut
    # h = 0: the plain blend
    _lib.check(lib.b200mdm_test_blend_handshake(_p(hres), _p(scale), _p(g16), B, T, d, s_off, halves, 0, None, None,
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    plain = (g16[:, :d].double() + g16[:, d:2 * d].double()).cpu()
    assert float(((plain - D).abs() / _bound(hres_c, sc_c, B, T, d, s_off, 0, lt, mt, halves, D, D)).max()) <= 1.0


# ------------------------------------------------------------------------------------------------ parity
@pytest.fixture(scope="module")
def small():
    c = gh.SMALL
    inp, shape, y = gh.small_inputs()
    cfg, diffusion = _model(c["L"], c["steps"], c["weights_seed"])
    return c, inp, shape, y, cfg, diffusion


def test_small_fixture_parity(golden, small):
    gold = golden("handshake_small.npz")
    c, inp, shape, y, cfg, diffusion = small
    hs = b200mdm.HandshakeSampleModel(cfg, c["h"])
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    t = torch.full((c["B"],), c["t_fwd"], dtype=torch.long, device="cuda")
    mask, motion = gh.inpaint_inputs(shape, c["inpaint_frames"])
    got = dict(
        fwd_guided=hs(xT, t, y=_y(inp, y)),
        fwd_unguided=b200mdm.HandshakeSampleModel(cfg.model, c["h"])(xT, t, y=_y(inp, y, scale=False)),
        ddpm=diffusion.p_sample_loop(hs, shape, noise=xT, clip_denoised=False, model_kwargs={"y": _y(inp, y)}, noise_tape=tape),
        ddim=diffusion.ddim_sample_loop(hs, shape, noise=xT, clip_denoised=False, eta=0.0, model_kwargs={"y": _y(inp, y)},
                                        noise_tape=tape),
        plms=diffusion.plms_sample_loop(hs, shape, noise=xT, clip_denoised=False, model_kwargs={"y": _y(inp, y)}, order=2),
        ddpm_inpaint=diffusion.p_sample_loop(hs, shape, noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={
            "y": _y(inp, y, inpainting_mask=mask.cuda(), inpainted_motion=motion.cuda())}))
    dec, ddiff = _model(c["L"], c["steps"], c["dec_weights_seed"], arch="trans_dec", emb_trans_dec=True,
                        text_encoder_type="clip")
    got["dec_ddpm"] = ddiff.p_sample_loop(b200mdm.HandshakeSampleModel(dec, c["h"]), shape, noise=xT, clip_denoised=False,
                                          model_kwargs={"y": _y(inp, y)}, noise_tape=tape)
    for k, v in got.items():
        e = rel_err(v, gold[k])
        print("%s: engine vs reference %.2e" % (k, e))
        assert e < (PLMS_TOL if k == "plms" else RTOL), (k, e)
    for k in ("ddpm", "ddim"):
        assert _dup_equal(got[k], y, c["h"], c["T"]), k
    print("PLMS final sample: handshake copies bit-identical: %s" % _dup_equal(got["plms"], y, c["h"], c["T"]))


def test_full_depth_fixture(golden):
    c = gh.C1
    inp, shape, y = gh.c1_inputs()
    cfg, diffusion = _model(c["L"], c["steps"], c["weights_seed"])
    out = diffusion.p_sample_loop(b200mdm.HandshakeSampleModel(cfg, c["h"]), shape, noise=inp["tape"][0].cuda(),
                                  clip_denoised=False, model_kwargs={"y": _y(inp, y)},
                                  noise_tape=torch.stack(inp["tape"][1:]).cuda())
    e = rel_err(out, golden("handshake_c1.npz")["ddpm"])
    print("full depth (L 8, 50 steps, T 196, 3 windows, h 20): engine vs reference %.2e" % e)
    assert e < RTOL
    assert _dup_equal(out, y, c["h"], c["T"])


@pytest.mark.parametrize("order", [1, 2])
def test_dpm_solver_vs_oracle(small, order):
    c, inp, shape, y, cfg, diffusion = small
    xT = inp["tape"][0]
    hs = b200mdm.HandshakeSampleModel(cfg, c["h"])
    out = diffusion.dpm_solver_sample_loop(hs, shape, noise=xT.cuda(), clip_denoised=False, model_kwargs={"y": _y(inp, y)},
                                           order=order)
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    den = ho.denoiser(po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], y["lengths"]), c["h"],
                      y["lengths"], y["motion_start"])
    with torch.no_grad():
        ref = do.dpm_loop(den, tabs, xT, order=order)
    e = rel_err(out, ref)
    print("DPM-Solver++ order %d: engine vs oracle %.2e" % (order, e))
    assert e < RTOL
    assert _dup_equal(out, y, c["h"], c["T"])


# ------------------------------------------------------------------------------------------------ the existing path
def test_h0_and_single_window_motions_are_the_plain_model(small):
    c, inp, shape, y, cfg, diffusion = small
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    yy = _y(inp, y)
    plain = diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": yy}, noise_tape=tape)
    h0 = diffusion.p_sample_loop(b200mdm.HandshakeSampleModel(cfg, 0), shape, noise=xT, clip_denoised=False,
                                 model_kwargs={"y": yy}, noise_tape=tape)
    singles = dict(yy, motion_start=torch.ones(c["B"], dtype=torch.bool, device="cuda"))
    alone = diffusion.p_sample_loop(b200mdm.HandshakeSampleModel(cfg, c["h"]), shape, noise=xT, clip_denoised=False,
                                    model_kwargs={"y": singles}, noise_tape=tape)
    assert torch.equal(h0, plain) and torch.equal(alone, plain)
    t = torch.full((c["B"],), 2, dtype=torch.long, device="cuda")
    assert torch.equal(b200mdm.HandshakeSampleModel(cfg, 0)(xT, t, y=yy), cfg(xT, t, y=yy))


def test_enotimpl_refusals(small):
    """DDIM inversion (a step and the loop) and the bound loop refuse handshakes at the C ABI."""
    c, inp, shape, y, cfg, diffusion = small
    B, T, steps = c["B"], c["T"], c["steps"]
    eng = cfg.model.engine()
    lib = eng.lib
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    eng.set_cond(B, T, _y(inp, y), True, torch.device("cuda"))
    # the tables first: a missing table is ESTATE before the refusal
    eng.set_schedule(diffusion.schedule_rows(0.0), diffusion._timestep_map(), key=None)
    eng.set_schedule_next(diffusion.schedule_next_rows())
    eng.set_schedule_vb(diffusion.schedule_vb_rows())
    eng.set_handshake(c["h"], B, T, _y(inp, y))
    x = inp["tape"][0].cuda()
    out = torch.empty_like(x)
    calls = {
        "reverse_step": lambda: lib.b200mdm_sample_step(eng.h, _lib.MODE_DDIM_REVERSE, 0, _p(x), None, 0, _p(out), None, s),
        "reverse": lambda: lib.b200mdm_ddim_reverse_loop_range(eng.h, 0, steps, _p(x), _p(out), 0, 1, s),
        "vb": lambda: lib.b200mdm_vb_loop_range(eng.h, steps - 1, steps, _p(x), None, 0, _lib.FLAG_PHILOX_NOISE, None, None, 1,
                                                s),
    }
    for name, call in calls.items():
        assert call() == _lib.ENOTIMPL, name
        assert b"handshakes" in lib.b200mdm_last_error(), name


# ------------------------------------------------------------------------------------------------ engine state
def test_engine_state_against_fresh_engines(small):
    c, inp, shape, y, cfg, diffusion = small
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    layout_a = _y(inp, y)
    layout_b = dict(layout_a, motion_start=torch.tensor([1, 0, 1, 0, 0], dtype=torch.bool, device="cuda"),
                    lengths=torch.tensor([24, 24, 20, 24, 18], device="cuda"))
    t = torch.full((c["B"],), 3, dtype=torch.long, device="cuda")

    def run(m, what, use_graph):
        if what == "hs_a":
            return diffusion.ddim_sample_loop(b200mdm.HandshakeSampleModel(m, c["h"]), shape, noise=xT, clip_denoised=False,
                                              model_kwargs={"y": layout_a}, noise_tape=tape, use_graph=use_graph)
        if what == "plain":
            return diffusion.ddim_sample_loop(m, shape, noise=xT, clip_denoised=False, model_kwargs={"y": layout_a},
                                              noise_tape=tape, use_graph=use_graph)
        if what == "hs_b":
            return diffusion.p_sample_loop(b200mdm.HandshakeSampleModel(m, c["h"]), shape, noise=xT, clip_denoised=False,
                                           model_kwargs={"y": layout_b}, noise_tape=tape, use_graph=use_graph)
        return m(xT, t, y=layout_a)
    for use_graph in (True, False):
        seq = [run(cfg, w, use_graph) for w in ("hs_a", "plain", "hs_b", "bare")]
        for w, got in zip(("hs_a", "plain", "hs_b", "bare"), seq):
            fresh, _ = _model(c["L"], c["steps"], c["weights_seed"])
            assert torch.equal(got, run(fresh, w, use_graph)), (w, use_graph)
            fresh.model.engine().close()


# ------------------------------------------------------------------------------------------------ sharding
def test_motion_aligned_shards_equal_the_batch(small):
    c, inp, shape, y, cfg, diffusion = small
    hs = b200mdm.HandshakeSampleModel(cfg, c["h"])
    kw = {"y": _y(inp, y)}
    full = diffusion.p_sample_loop(hs, shape, clip_denoised=False, model_kwargs=kw, noise_seed=7)
    parts = []
    for lo, hi in ((0, 3), (3, 5)):
        local = parallel.shard_model_kwargs(kw, lo, hi)
        parts.append(diffusion.p_sample_loop(hs, (hi - lo,) + tuple(shape[1:]), clip_denoised=False, model_kwargs=local,
                                             noise_seed=7, sample_index_base=lo))
    assert torch.equal(torch.cat(parts), full)


# ------------------------------------------------------------------------------------------------ headline shape
def test_headline_64_windows_ddim50():
    L, steps, T, h, motions, per = 8, 50, 196, 20, 8, 8
    B = motions * per
    lengths = [196 if k % 3 else 176 for k in range(B)]
    starts = [k % per == 0 for k in range(B)]
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=63, lengths=lengths, scale=2.5)
    y = dict(mask=inp["mask"], lengths=inp["lengths"], text_embed=inp["text_embed"],
             motion_start=torch.tensor(starts, dtype=torch.bool))
    cfg, diffusion = _model(L, steps, 1)
    out = diffusion.ddim_sample_loop(b200mdm.HandshakeSampleModel(cfg, h), (B, 263, 1, T), noise=inp["tape"][0].cuda(),
                                     clip_denoised=False, eta=0.0, model_kwargs={"y": _y(inp, y)},
                                     noise_tape=torch.stack(inp["tape"][1:]).cuda())
    assert _dup_equal(out, y, h, T)
    m = slice(per, 2 * per)                                                     # motion 1, windows 8 .. 15
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=L, seed=1), L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    ln, ms = y["lengths"][m], y["motion_start"][m]
    den = ho.denoiser(po.enc_denoiser(W, list(range(steps)), inp["text_embed"][:, m], inp["scale"][m], ln), h, ln, ms)
    with torch.no_grad():
        ref = deo.sample_loop(den, tabs, [t[m] for t in inp["tape"]], sampler="ddim")
    e = rel_err(out[m], ref)
    print("headline (64 windows, 8 motions of 8, h 20, DDIM 50): motion 1 vs the fp32 oracle %.2e" % e)
    assert e < RTOL
