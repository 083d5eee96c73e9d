"""GPU: the CLIP-conditioned decoder with a timestep token (arch='trans_dec', text_encoder_type='clip',
emb_trans_dec=True; the humanml-decoder-with-emb checkpoint).

  * its two kernels against fp64: the per-step cross-attention rows (cross_rows_kernel and the per-loop / per-weight-load
    GEMVs behind it) and the row-bias LayerNorm, each with a per-element bound derived from its fp32 arithmetic and
    mutants (plausible bugs) that must exceed the bound at least 8-fold;
  * parity with the reference's fixtures (tests/golden/dec_emb_*.npz) and, at the headline shape and over 1000 steps,
    with the fp32 oracle following a few samples; PLMS and DDIM inversion against the oracle; the Philox loop split
    into two batch halves.
Tolerance: 1e-3 relative (Frobenius)."""
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from conftest import default_args, rel_err

pytestmark = pytest.mark.gpu
RTOL = 1e-3
U = 2.0 ** -24
syn = importlib.import_module("motion-diffusion-model_b200.synthetic")


def _dec(layers, steps, seed, sd=None, **over):
    args = default_args(layers=layers, diffusion_steps=steps, arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True,
                        **over)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    if sd is None:
        sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=layers, cond_dim=512, seed=seed,
                                      target_encoder=over.get("multi_encoder_type") if over.get("multi_target_cond") else None)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion, sd


def _y(inp, scale=True, dev="cuda", **extra):
    y = dict(mask=inp["mask"].to(dev), lengths=inp["lengths"].to(dev), text_embed=inp["text_embed"].to(dev), **extra)
    if scale:
        y["scale"] = inp["scale"].to(dev)
    return y


def _tape(inp):
    return inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()


# ------------------------------------------------------------------------------------------------ kernels vs fp64
def _lin_err(W, x, b, Ex):
    """First-order bound of the fp32 y = W x + b of small_linear_kernel (per lane a chain of K/32 fmas, a 5-level
    shuffle tree, the bias add: < 24 roundings per output) from x carrying the error bound Ex."""
    aW = W.abs()
    carried = Ex @ aW.T if torch.is_tensor(Ex) else 0.0
    return carried + 24 * U * (x.abs() @ aW.T + (b.abs() if b is not None else 0))


def _cross_rows64(sd, L, clip, t, B, wrong_layer=False, drop_bv=False, uncond_text=False):
    """fp64 c [L, 2B, d] of c_l[b'] = W_o,l (W_v,l (textproj[b'] + temb[t]) + b_v,l) + b_o,l, and its error bound."""
    W = {k: v.double() for k, v in sd.items()}
    d = 512
    pe = b200mdm.model.mdm.positional_table(5000, d).double()[t][None]
    h1 = pe @ W["embed_timestep.time_embed.0.weight"].T + W["embed_timestep.time_embed.0.bias"]
    s = torch.nn.functional.silu(h1)
    temb = s @ W["embed_timestep.time_embed.2.weight"].T + W["embed_timestep.time_embed.2.bias"]
    E_h = _lin_err(W["embed_timestep.time_embed.0.weight"], pe, W["embed_timestep.time_embed.0.bias"], 0)
    E_s = 1.1 * E_h + 8 * U * s.abs()
    E_t = _lin_err(W["embed_timestep.time_embed.2.weight"], s, W["embed_timestep.time_embed.2.bias"], E_s)
    c64 = clip.double()
    pc = c64 @ W["embed_text.weight"].T + W["embed_text.bias"]
    E_pc = _lin_err(W["embed_text.weight"], c64, W["embed_text.bias"], 0)
    pu = pc if uncond_text else W["embed_text.bias"].expand(B, d)
    p = torch.cat([pc, pu])
    E_p = torch.cat([E_pc, E_pc if uncond_text else torch.zeros(B, d, dtype=torch.float64)])
    out, bound = [], []
    for l in range(L):
        q = "seqTransDecoder.layers.%d." % l
        o = "seqTransDecoder.layers.%d." % ((l + 1) % L if wrong_layer else l)
        Wv, bv = W[q + "multihead_attn.in_proj_weight"][2 * d:], W[q + "multihead_attn.in_proj_bias"][2 * d:]
        Wo, bo = W[o + "multihead_attn.out_proj.weight"], W[o + "multihead_attn.out_proj.bias"]
        v = (p + temb) @ Wv.T + (0 if drop_bv else bv)
        c = v @ Wo.T + bo
        out.append(c)
        # the engine's split: cb = W_o (W_v p + b_v) + b_o per loop, ct = W_o (W_v temb) per weight load, c = cb + ct
        ub, ut = p @ Wv.T + bv, temb @ Wv.T
        E_cb = _lin_err(Wo, ub, bo, _lin_err(Wv, p, bv, E_p))
        E_ct = _lin_err(Wo, ut, None, _lin_err(Wv, temb, None, E_t))
        bound.append(E_cb + E_ct + 2 * U * (c.abs() + (ub @ Wo.T).abs() + (ut @ Wo.T).abs()) + 1e-30)
    return torch.stack(out), torch.stack(bound)


def test_cross_rows_vs_fp64():
    L, B, T, t = 2, 3, 24, 37
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=41)
    for l in range(L):   # value biases of the size of the other terms, so that dropping them is visible
        k = "seqTransDecoder.layers.%d.multihead_attn.in_proj_bias" % l
        sd[k] = sd[k] * 25.0
    cfg, model, diffusion, _ = _dec(L, 50, 0, sd=sd)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=1, seed=42)
    eng = model.engine()
    eng.set_cond(B, T, _y(inp), True, torch.device("cuda"))
    got = eng.test_cross_rows(t, 2, "cuda").double().cpu()
    clip = inp["text_embed"][0]
    want, bound = _cross_rows64(sd, L, clip, t, B)
    ratio = ((got - want).abs() / bound).max().item()
    mutants = {"b_v dropped": _cross_rows64(sd, L, clip, t, B, drop_bv=True)[0],
               "out-projection of the wrong layer": _cross_rows64(sd, L, clip, t, B, wrong_layer=True)[0],
               "unconditional half given the text": _cross_rows64(sd, L, clip, t, B, uncond_text=True)[0]}
    mr = {k: ((m - want).abs() / bound).max().item() for k, m in mutants.items()}
    print("cross rows: error / bound %.3g (max |c| %.3g, max bound %.3g); mutants: %s" % (
        ratio, want.abs().max().item(), bound.max().item(), ", ".join("%s %.3g" % kv for kv in mr.items())))
    assert ratio <= 1.0
    for k, v in mr.items():
        assert v >= 8.0, k


def _ln64(v, gamma, beta):
    mu = v.mean(-1, keepdim=True)
    var = ((v - mu) ** 2).mean(-1, keepdim=True)
    return (v - mu) / torch.sqrt(var + 1e-5) * gamma + beta, mu, var


def test_row_bias_layernorm_vs_fp64():
    from b200mdm import _lib
    lib = _lib.load()
    B, S, d = 3, 37, 512
    Bp, M = 2 * B, 2 * B * S
    g = torch.Generator().manual_seed(7)
    val = torch.randn(M, d, generator=g) * 1.5 + torch.randn(M, 1, generator=g)
    hi = val.half()
    lo = (val - hi.float()).half()
    h = torch.cat([hi, lo], 1).cuda()
    c = torch.randn(Bp, d, generator=g).cuda()
    g2, b2 = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    g3, b3 = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    g2d, b2d = g2.cuda(), b2.cuda()   # (named: a temporary's memory could be reused before the kernel reads it)
    _lib.check(lib.b200mdm_test_row_bias_ln(h.data_ptr(), c.data_ptr(), g2d.data_ptr(), b2d.data_ptr(), M, S,
                                            torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    h = h.cpu()
    got = h[:, :d].double() + h[:, d:].double()
    x = hi.double() + lo.double()
    crow = c.cpu().double()[torch.arange(M) // S]
    v = x + crow
    want, mu, var = _ln64(v, g2.double(), b2.double())
    # fp32 arithmetic: v = (hi + lo) + c rounds once (hi + lo is exact); the sums are 16-term chains + a 5-level tree;
    # rsqrtf <= 2 ulp; y = (v - mean) rstd gamma + beta four roundings; hi + lo keeps y to 2^-22 (2^-25 absolute)
    av = v.abs()
    e_v = U * av
    e_mu = U * av.max(-1, keepdim=True).values + 22 * U * av.mean(-1, keepdim=True)
    e_var = 2 * (e_mu + e_v.max(-1, keepdim=True).values) * (v - mu).abs().mean(-1, keepdim=True) + 24 * U * var
    rstd = 1 / torch.sqrt(var + 1e-5)
    e_rstd = rstd * (0.5 * e_var / (var + 1e-5) + 4 * U)
    xhat = (v - mu) * rstd
    y_abs = want.abs()
    bound = 2 * (g2.double().abs() * (rstd * (e_v + e_mu) + (v - mu).abs() * e_rstd) +
                 6 * U * (g2.double().abs() * xhat.abs() + b2.double().abs()) + 2.0 ** -22 * y_abs + 2.0 ** -25)
    ratio = ((got - want).abs() / bound).max().item()
    swap = torch.cat([torch.arange(B, Bp), torch.arange(0, B)])
    mutants = {"c of the other CFG half": _ln64(x + c.cpu().double()[swap][torch.arange(M) // S], g2.double(), b2.double())[0],
               "c added after the LayerNorm": _ln64(x, g2.double(), b2.double())[0] + crow,
               "norm3 parameters": _ln64(v, g3.double(), b3.double())[0]}
    mr = {k: ((m - want).abs() / bound).max().item() for k, m in mutants.items()}
    print("row-bias LayerNorm: error / bound %.3g; mutants: %s" % (ratio, ", ".join("%s %.3g" % kv for kv in mr.items())))
    assert ratio <= 1.0
    for k, r in mr.items():
        assert r >= 8.0, k


# ------------------------------------------------------------------------------------------------ parity
def test_vs_reference_golden_small(golden):
    g = golden("dec_emb_small.npz")
    L, steps, B, T = 2, 4, 3, 24
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=15, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 7.5]))
    x, tape = _tape(inp)
    shape = (B, 263, 1, T)
    t = torch.full((B,), 2, dtype=torch.long, device="cuda")
    motion = torch.from_numpy(g["inpaint_motion"]).cuda()
    imask = torch.zeros(shape, dtype=torch.bool, device="cuda")
    imask[..., :8] = True
    got = {}
    cfg, model, diffusion, _ = _dec(L, steps, 9)
    got["fwd_cond"] = model(x, t, y=_y(inp, False))
    got["fwd_uncond"] = model(x, t, y=_y(inp, False, uncond=True))
    got["fwd_cfg"] = cfg(x, t, y=_y(inp))
    kw = dict(noise=x, clip_denoised=False, noise_tape=tape)
    got["ddpm"] = diffusion.p_sample_loop(cfg, shape, model_kwargs={"y": _y(inp)}, **kw)
    got["ddim_eta0"] = diffusion.ddim_sample_loop(cfg, shape, eta=0.0, model_kwargs={"y": _y(inp)}, **kw)
    got["ddpm_inpaint"] = diffusion.p_sample_loop(cfg, shape, model_kwargs={
        "y": _y(inp, inpainting_mask=imask, inpainted_motion=motion)}, **kw)
    cfg, model, diffusion, _ = _dec(L, steps, 9, mask_frames=False)
    got["nomask_fwd_cfg"] = cfg(x, t, y=_y(inp))
    got["nomask_ddpm"] = diffusion.p_sample_loop(cfg, shape, model_kwargs={"y": _y(inp)}, **kw)
    cfg, model, diffusion, _ = _dec(L, steps, 9, multi_target_cond=True, multi_encoder_type="single", target_enc_layers=1)
    tg = syn.synthetic_target_inputs(B, seed=5)
    ty = dict(target_cond=tg["target_cond"].cuda(), target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    got["target_fwd_cfg"] = cfg(x, t, y=_y(inp, **ty))
    got["target_ddpm"] = diffusion.p_sample_loop(cfg, shape, model_kwargs={"y": _y(inp, **ty)}, **kw)
    for k, v in got.items():
        e = rel_err(v, g[k])
        print("%-16s %.3e" % (k, e))
        assert e < RTOL, k


def test_vs_reference_golden_c1(golden):
    g = golden("dec_emb_c1.npz")
    cfg, _, diffusion, _ = _dec(8, 50, 0)
    inp = b200mdm.synthetic_inputs(1, nframes=196, steps=50, seed=10)
    x, tape = _tape(inp)
    out = diffusion.p_sample_loop(cfg, (1, 263, 1, 196), noise=x, clip_denoised=False, model_kwargs={"y": _y(inp)},
                                  noise_tape=tape)
    e = rel_err(out, g["sample"])
    print("decoder c1 (L=8, T=196, 50 steps, CFG 2.5) vs reference: %.3e" % e)
    assert e < RTOL


def test_c2_shape_b64_50_steps():
    """The headline shape: B=64, 196 frames, 50 steps, CFG 2.5, L=8; the fp32 oracle follows 3 samples."""
    from oracle import dec_emb_oracle as deo, mdm_oracle as mo, schedule_oracle as so
    B, T, steps = 64, 196, 50
    cfg, _, diffusion, sd = _dec(8, steps, 0)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, lengths=[196 - (b * 7) % 150 for b in range(B)])
    x, tape = _tape(inp)
    out = diffusion.p_sample_loop(cfg, (B, 263, 1, T), noise=x, clip_denoised=False, model_kwargs={"y": _y(inp)}, noise_tape=tape)
    assert torch.isfinite(out).all()
    idx = [0, 31, 63]
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = deo.denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    ref = deo.sample_loop(f, tabs, [t[idx] for t in inp["tape"]])
    e = rel_err(out[idx].cpu(), ref)
    print("decoder B=64 x 50 steps x CFG 2.5: relative error %.3e" % e)
    assert e < RTOL


class _LazyTape:
    """tape[0] = x_T, tape[1+k] = eps of the k-th step, from the engine's Philox stream for the followed samples."""

    def __init__(self, eng, idx, shape1, seed, n_steps):
        self.eng, self.idx, self.shape1, self.seed, self.n = eng, idx, shape1, seed, n_steps

    def __getitem__(self, k):
        step_id = -1 if k == 0 else self.n - k
        return torch.cat([self.eng.philox_normal((1,) + self.shape1, self.seed, g, step_id, "cuda") for g in self.idx]).cpu()


def test_1000_step_schedule_vs_oracle():
    """The checkpoint's own 1000-step schedule through the fused loop (Philox noise); the oracle follows 2 samples."""
    from oracle import dec_emb_oracle as deo, mdm_oracle as mo, schedule_oracle as so
    B, T, steps, seed = 8, 196, 1000, 91
    cfg, model, diffusion, sd = _dec(8, steps, 0)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=1, seed=12, lengths=[196, 150, 120, 90, 196, 60, 33, 196])
    out = diffusion.p_sample_loop(cfg, (B, 263, 1, T), clip_denoised=False, model_kwargs={"y": _y(inp)}, noise_seed=seed)
    idx = [1, 6]
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = deo.denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    ref = deo.sample_loop(f, tabs, _LazyTape(model.engine(), idx, (263, 1, T), seed, steps))
    e = rel_err(out[idx].cpu(), ref)
    print("decoder 1000 steps: relative error %.3e" % e)
    assert e < RTOL


def test_plms_and_ddim_inversion_vs_oracle():
    from oracle import dec_emb_oracle as deo, mdm_oracle as mo, plms_oracle as po, reverse_oracle as ro, schedule_oracle as so
    L, steps, B, T = 2, 20, 3, 40
    cfg, _, diffusion, sd = _dec(L, steps, 9)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=17, lengths=[40, 31, 9], scale=torch.tensor([2.5, 1.0, 2.5]))
    x = inp["tape"][0]
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = deo.denoiser(W, list(range(steps)), inp["text_embed"], inp["scale"], inp["lengths"])
    kw = dict(clip_denoised=False, model_kwargs={"y": _y(inp)})
    for order in (2, 4):
        out = diffusion.plms_sample_loop(cfg, (B, 263, 1, T), noise=x.cuda(), order=order, **kw)
        e = rel_err(out, po.plms_loop(f, tabs, x, order=order))
        print("decoder PLMS order %d, %d steps: %.3e" % (order, steps, e))
        assert e < RTOL, order
    out = diffusion.ddim_reverse_sample_loop(cfg, x.cuda(), **kw)
    e = rel_err(out, ro.reverse_loop(f, tabs, x))
    print("decoder DDIM inversion, %d steps: %.3e" % (steps, e))
    assert e < RTOL


def test_philox_loop_split_into_batch_halves_is_bit_identical():
    L, steps, B, T, seed = 2, 10, 6, 33, 777
    cfg, _, diffusion, _ = _dec(L, steps, 9)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=1, seed=21, lengths=[33, 30, 20, 9, 2, 1])
    y = _y(inp)
    full = diffusion.p_sample_loop(cfg, (B, 263, 1, T), clip_denoised=False, model_kwargs={"y": y}, noise_seed=seed)
    parts = []
    for lo, hi in ((0, 3), (3, 6)):
        ys = dict(mask=y["mask"][lo:hi], lengths=y["lengths"][lo:hi], text_embed=y["text_embed"][:, lo:hi].contiguous(),
                  scale=y["scale"][lo:hi])
        parts.append(diffusion.p_sample_loop(cfg, (hi - lo, 263, 1, T), clip_denoised=False, model_kwargs={"y": ys},
                                             noise_seed=seed, sample_index_base=lo))
    assert torch.equal(torch.cat(parts), full)
