"""GPU: every stage of the engine's own forward, layer by layer, through b200mdm_test_forward_taps.

The kernel-level tests reach each kernel through its b200mdm_test_* hook, which builds its own tensor maps over
contiguous buffers.  The step wires the same kernels with its own maps, pitches, layer offsets and CFG halves.  Here:
(a) each tapped stage output equals, bit for bit, the same kernel's hook fed with the tapped input of that stage and the
state-dict weights converted by torch (fp16 round-to-nearest, [W | W] where the DiP engine keeps [hi | lo]
activations); the valid-key counts and the memory mask are derived from y, not read from the engine;
(b) for each stage at least one wiring mutant pushed through the same hook differs from the engine somewhere;
(c) the kernels without a hook (token 0, the conditioning rows, the timestep-embedding rows, the DiP memory rows) hold
per-element bounds derived from their fp32 arithmetic against fp64, and their mutants exceed them by 8x.
Then the shape envelope (S = 64 / 65 / 208 / 209 / 256) through the engine against the fp32 oracle, and the step with
programmatic dependent launch off (B200MDM_PDL=0, in a child process) against the step with it on."""
import ctypes
import importlib
import os
import subprocess
import sys
import tempfile
from types import SimpleNamespace

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":   # the PDL-off child process (test_pdl_off_equals_pdl_on)
    sys.path[:0] = [os.path.dirname(HERE), HERE]

import b200mdm  # noqa: E402
from conftest import default_args  # noqa: E402

pytestmark = pytest.mark.gpu
syn = importlib.import_module("motion-diffusion-model_b200.synthetic")

MUTANT_MARGIN = 8.0
U32 = 2.0 ** -24
D, FF = 512, 1024
F64 = torch.float64


def _lib():
    from b200mdm import _lib as L
    return L, L.load()


def _p(t, byte_off=0):
    return ctypes.c_void_p(t.data_ptr() + byte_off) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ the hooks
def gemm16(a, w16, bias, act):
    """b200mdm_test_gemm_f16, 128 x 128 tiles (the step's projection kernel)."""
    L, lib = _lib()
    M, K = a.shape
    out = torch.empty(M, w16.shape[0], device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_gemm_f16(_p(a), _p(w16), _p(bias), _p(out), M, w16.shape[0], K, act, 128, _stream()))
    return out


def gemm_epi(a, w16, bias, epi):
    L, lib = _lib()
    M, K = a.shape
    N = w16.shape[0]
    out = torch.empty(M, 2 * N if epi == 0 else N, device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_gemm_epi(_p(a), _p(w16), _p(bias), _p(out), M, N, K, epi, _stream()))
    return out


def attention(qkv, kvlen, n, S, wide):
    L, lib = _lib()
    out = torch.empty(n * S, (2 if wide else 1) * D, device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_attention(_p(qkv), _p(out), _p(kvlen), n, S, D, int(wide), _stream()))
    return out


def resid_ln(a, w16, bias, gamma, beta, hres):
    """b200mdm_test_gemm_resid_ln on a copy of hres."""
    L, lib = _lib()
    h = hres.clone()
    L.check(lib.b200mdm_test_gemm_resid_ln(_p(a), _p(w16), _p(bias), _p(gamma), _p(beta), _p(h), a.shape[0], a.shape[1],
                                           _stream()))
    return h


def cross_attention(q, kv, col, ld, mask, n, S, Mt):
    """b200mdm_test_cross_attention on kv's columns [col, col + 2d) (row pitch ld); returns columns [0, d) of the output."""
    L, lib = _lib()
    out = torch.zeros(n * S, 2 * D, device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_cross_attention(_p(q), _p(kv, 2 * col), _p(mask), _p(out), n, S, Mt, ld, _stream()))
    return out[:, :D]


def row_bias_ln(hres, c, gamma, beta, S):
    L, lib = _lib()
    h = hres.clone()
    L.check(lib.b200mdm_test_row_bias_ln(_p(h), _p(c.contiguous()), _p(gamma), _p(beta), h.shape[0], S, _stream()))
    return h


def embed(x, w_in, b_in, pe, s_off, halves):
    L, lib = _lib()
    B, JF, T = x.shape
    out = torch.empty(halves * B * (T + s_off), 2 * D, device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_embed(_p(x), _p(w_in), _p(b_in), _p(pe), _p(out), B, JF, T, D, s_off, halves, _stream()))
    return out


def out_x0(hres, scale, w_out, b_out, x, s_off, halves):
    """b200mdm_test_out_step in mode X0: the model output."""
    L, lib = _lib()
    B, JF, T = x.shape
    xo, pred = torch.empty_like(x), torch.empty_like(x)
    L.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w_out), _p(b_out), _p(x), None, None, L.MODE_X0, 0, None,
                                      None, _p(xo), _p(pred), B, JF, T, D, s_off, halves, _stream()))
    return xo


def f16(w, kw=1):
    """The state-dict weight as the engine converts it: fp16 RNE, [W | W] along K for kw = 2."""
    h = w.half()
    return torch.cat([h, h], 1).contiguous() if kw == 2 else h.contiguous()


# ------------------------------------------------------------------------------------------------ model cases
def build(kind, B, T, L, seed, guided, lengths=None, scale=None, Mt=16, ctx=20, target=None, dataset=None):
    """A loaded engine with its conditioning set, and everything the checks need: weights (the model's own state dict,
    fp32 on the GPU), inputs, y and the shape of the step.  dataset="kit": a text model (trans_enc or DiP) at KIT's 251
    features."""
    over = dict(layers=L, diffusion_steps=50)
    ds, sdkw, njoints, nfeats = {}, {}, 263, 1
    if kind == "a2m":
        over.update(dataset="humanact12", cond_mask_prob=0.0)
        ds, sdkw, njoints, nfeats = dict(num_actions=12), dict(input_feats=150, cond_mode="action", num_actions=12), 25, 6
    elif kind == "dip":
        over.update(arch="trans_dec", text_encoder_type="bert", context_len=ctx, pred_len=T)
        sdkw = dict(arch="trans_dec", cond_dim=768)
    elif kind == "dec_emb":
        over.update(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
        sdkw = dict(arch="trans_dec", cond_dim=512)
    if dataset == "kit":
        over.update(dataset="kit")
        sdkw["input_feats"], njoints = 251, 251
    if target:
        over.update(multi_target_cond=True, multi_encoder_type=target, target_enc_layers=1)
        sdkw.update(target_encoder=target, target_enc_layers=1)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace(**ds)))
    sd = syn.synthetic_state_dict(num_layers=L, seed=seed, **sdkw)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    inp = syn.synthetic_inputs(B, njoints=njoints, nfeats=nfeats, nframes=T, steps=3, seed=seed + 1, lengths=lengths,
                               scale=scale if scale is not None else 2.5)
    y = dict(mask=inp["mask"], lengths=inp["lengths"])
    if guided:
        y["scale"] = inp["scale"]
    c = SimpleNamespace(kind=kind, B=B, T=T, L=L, guided=guided, halves=2 if guided else 1, Mt=0, ctx=0, g=None,
                        model=model, diffusion=diffusion, sd=sd, inp=inp, shape=(B, njoints, nfeats, T), JF=njoints * nfeats)
    if kind in ("enc", "dec_emb"):
        y["text_embed"] = inp["text_embed"]
    elif kind == "a2m":
        y["action"] = torch.arange(B).remainder(12).view(B, 1)
    elif kind == "dip":
        enc, tmask, prefix = syn.synthetic_dip_inputs(B, Mt, ctx, njoints=njoints, seed=seed + 2)
        y["text_embed"], c.Mt, c.ctx = (enc, tmask), Mt, ctx
        if ctx:
            y["prefix"] = prefix
    if target:
        tg = syn.synthetic_target_inputs(B, seed=seed + 3)
        y.update(target_cond=tg["target_cond"], target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    c.y = {k: (v.cuda() if torch.is_tensor(v) else tuple(u.cuda() for u in v) if isinstance(v, tuple) else v)
           for k, v in y.items()}
    c.eng = model.engine()
    c.eng.set_cond(B, T, c.y, guided, "cuda")
    if target:
        from b200mdm.engine import canonical_target
        tc, valid = canonical_target(c.y, B, c.eng.target_joint_names)
        c.g = c.eng.test_target(tc.cuda(), valid)
    c.W = {k: v.detach().float().cuda().contiguous() for k, v in model.state_dict().items()}
    c.pe = model.sequence_pos_encoder.pe.detach().reshape(-1, D).float().cuda().contiguous()   # (a buffer, not in the state dict)
    c.pre = "seqTransDecoder.layers." if kind in ("dip", "dec_emb") else "seqTransEncoder.layers."
    c.dec, c.dip = kind in ("dip", "dec_emb"), kind == "dip"
    c.kw = 2 if c.dip else 1
    c.s_off = ctx if kind == "dip" else 1
    c.S = T + c.s_off
    c.Bp = c.halves * B
    c.M = c.Bp * c.S
    c.x = inp["tape"][0].cuda()
    c.ts = (torch.arange(B) * 7 + 3) % 50           # distinct per-sample model timesteps
    c.scale = c.y["scale"].float().contiguous() if guided else None
    # valid keys per sample as the reference derives them (model/mdm.py:241-247): the tokens before the frames, then
    # y['lengths'] frames; a memory mask from the text padding mask (True = padding), both repeated for the CFG halves
    ln = c.y["mask"].reshape(B, -1).sum(-1).int() if T > 1 else torch.full((B,), T, dtype=torch.int32, device="cuda")
    c.kvlen = (ln + c.s_off).clamp(max=c.S).repeat(c.halves).int().contiguous()
    if c.dip:
        c.memmask = c.y["text_embed"][1].to(torch.uint8).repeat(c.halves, 1).contiguous()
    return c


def lw(c, l, name):
    return c.W[c.pre + "%d." % l + name]


class Record:
    """Stage results of one case: bit-identity failures and mutants that fail to differ, asserted at the end."""

    def __init__(self, title):
        self.title, self.bad = title, []
        print("\n== %s" % title)

    def same(self, name, got, ref):
        g, r = got.contiguous(), ref.contiguous()
        it = torch.int16 if g.dtype == torch.float16 else torch.int32
        n = int((g.view(it) != r.view(it)).sum())
        print("  %-44s %d differing elements" % (name, n))
        if n or g.shape != r.shape:
            self.bad.append("%s differs from its hook in %d elements" % (name, n))

    def teeth(self, name, got, mut):
        g, m = got.contiguous(), mut.contiguous()
        it = torch.int16 if g.dtype == torch.float16 else torch.int32
        n = int((g.view(it) != m.view(it)).sum())
        print("    mutant %-37s %d differing elements" % (name, n))
        if n == 0:
            self.bad.append("mutant %s is indistinguishable" % name)

    def bound(self, name, err, bound, mutants):
        r = float((err / bound).max())
        msg = "  %-44s error / bound = %.3g" % (name, r)
        print(msg)
        if not (torch.isfinite(err).all() and r <= 1.0):
            self.bad.append("%s: error %.3g x its bound" % (name, r))
        for mname, merr in mutants.items():
            mr = float((merr / bound).max())
            print("    mutant %-37s error / bound = %.3g" % (mname, mr))
            if not mr >= MUTANT_MARGIN:
                self.bad.append("%s: mutant %s only %.3g x the bound" % (name, mname, mr))

    def done(self):
        assert not self.bad, "%s:\n  %s" % (self.title, "\n  ".join(self.bad))


# ------------------------------------------------------------------------------------------------ (a) + (b): hooks
def check_layer(c, l, t, out, rec):
    """Every stage of layer l against its hook; t: the taps of a forward tapped at l."""
    other = l + 1 if l + 1 < c.L else l - 1      # "the weights of layer l +- 1"
    S, M, kw, d = c.S, c.M, c.kw, D
    W = lambda n, k=1, ll=l: f16(lw(c, ll, n), k)   # noqa: E731
    V = lambda n, ll=l: lw(c, ll, n)                # noqa: E731
    h_in = t["L_IN"]
    # QKV projection: the hi half of the residual stream, K = d
    a = h_in[:, :d].contiguous()
    rec.same("L%d QKV GEMM" % l, t["L_QKV"], gemm16(a, W("self_attn.in_proj_weight"), V("self_attn.in_proj_bias"), 0))
    rec.teeth("L%d QKV: weights of layer %d" % (l, other), t["L_QKV"],
              gemm16(a, W("self_attn.in_proj_weight", ll=other), V("self_attn.in_proj_bias", other), 0))
    # self-attention core
    rec.same("L%d self-attention" % l, t["L_ATT"], attention(t["L_QKV"], c.kvlen, c.Bp, S, c.dip))
    rec.teeth("L%d attention: kvlen + 1" % l, t["L_ATT"],
              attention(t["L_QKV"], (c.kvlen + 1).clamp(max=S).int().contiguous(), c.Bp, S, c.dip))
    # out-projection + LN1 (K = kw d: the [hi | lo] attention output of DiP against [W | W])
    wo = W("self_attn.out_proj.weight", kw)
    ln1 = resid_ln(t["L_ATT"], wo, V("self_attn.out_proj.bias"), V("norm1.weight"), V("norm1.bias"), h_in)
    rec.same("L%d out-proj + LN1" % l, t["L_LN1"], ln1)
    rec.teeth("L%d out-proj: weights of layer %d" % (l, other), t["L_LN1"],
              resid_ln(t["L_ATT"], W("self_attn.out_proj.weight", kw, other), V("self_attn.out_proj.bias", other),
                       V("norm1.weight", other), V("norm1.bias", other), h_in))
    if c.dip:
        rec.teeth("L%d out-proj: hi half only" % l, t["L_LN1"],
                  resid_ln(t["L_ATT"][:, :d].contiguous(), W("self_attn.out_proj.weight"), V("self_attn.out_proj.bias"),
                           V("norm1.weight"), V("norm1.bias"), h_in))
    h_ffn = t["L_LN1"]
    if c.dip:
        # cross-attention: Q GEMM on the hi half, the core on this layer's K | V columns, out-proj + LN2 on the hi half
        a = t["L_LN1"][:, :d].contiguous()
        wq, bq = lw(c, l, "multihead_attn.in_proj_weight")[:d], lw(c, l, "multihead_attn.in_proj_bias")[:d].contiguous()
        rec.same("L%d cross Q GEMM" % l, t["L_QC"], gemm16(a, f16(wq), bq, 0))
        wq_o = lw(c, other, "multihead_attn.in_proj_weight")[:d]
        rec.teeth("L%d cross Q: weights of layer %d" % (l, other), t["L_QC"],
                  gemm16(a, f16(wq_o), lw(c, other, "multihead_attn.in_proj_bias")[:d].contiguous(), 0))
        ld = c.L * 2 * d
        xat = t["L_XATT"][:, :d]
        rec.same("L%d cross-attention core" % l, xat,
                 cross_attention(t["L_QC"], t["KVC16"], l * 2 * d, ld, c.memmask, c.Bp, S, c.Mt))
        prev = l - 1 if l > 0 else l + 1
        rec.teeth("L%d cross core: K/V of layer %d" % (l, prev), xat,
                  cross_attention(t["L_QC"], t["KVC16"], prev * 2 * d, ld, c.memmask, c.Bp, S, c.Mt))
        rec.teeth("L%d cross core: memory mask ignored" % l, xat,
                  cross_attention(t["L_QC"], t["KVC16"], l * 2 * d, ld, torch.zeros_like(c.memmask), c.Bp, S, c.Mt))
        a = xat.contiguous()
        rec.same("L%d cross out-proj + LN2" % l, t["L_LN2"],
                 resid_ln(a, W("multihead_attn.out_proj.weight"), V("multihead_attn.out_proj.bias"), V("norm2.weight"),
                          V("norm2.bias"), t["L_LN1"]))
        rec.teeth("L%d cross out-proj: weights of layer %d" % (l, other), t["L_LN2"],
                  resid_ln(a, W("multihead_attn.out_proj.weight", ll=other), V("multihead_attn.out_proj.bias", other),
                           V("norm2.weight", other), V("norm2.bias", other), t["L_LN1"]))
        h_ffn = t["L_LN2"]
    elif c.dec:
        # the CLIP decoder's one-token cross-attention: h <- LN2(h + c_l[sample])
        rows = t["CROSS_C"]
        rec.same("L%d row-bias LN2" % l, t["L_LN2"], row_bias_ln(t["L_LN1"], rows[l], V("norm2.weight"), V("norm2.bias"), S))
        prev = l - 1 if l > 0 else l + 1
        rec.teeth("L%d row-bias LN2: cross rows of layer %d" % (l, prev), t["L_LN2"],
                  row_bias_ln(t["L_LN1"], rows[prev], V("norm2.weight"), V("norm2.bias"), S))
        rec.teeth("L%d row-bias LN2: norm2 of layer %d" % (l, other), t["L_LN2"],
                  row_bias_ln(t["L_LN1"], rows[l], V("norm2.weight", other), V("norm2.bias", other), S))
        h_ffn = t["L_LN2"]
    # FFN-up (GELU): DiP reads the whole [hi | lo] stream against [W | W] and writes [hi | lo]
    if c.dip:
        ffn = gemm_epi(h_ffn, W("linear1.weight", 2), V("linear1.bias"), 0)
        mut_l = gemm_epi(h_ffn, W("linear1.weight", 2, other), V("linear1.bias", other), 0)
        mut_hi = gemm_epi(h_ffn[:, :d].contiguous(), W("linear1.weight"), V("linear1.bias"), 0)
    else:
        a = h_ffn[:, :d].contiguous()
        ffn = gemm16(a, W("linear1.weight"), V("linear1.bias"), 1)
        mut_l, mut_hi = gemm16(a, W("linear1.weight", ll=other), V("linear1.bias", other), 1), None
    rec.same("L%d FFN-up" % l, t["L_FFN"], ffn)
    rec.teeth("L%d FFN-up: weights of layer %d" % (l, other), t["L_FFN"], mut_l)
    if mut_hi is not None:
        rec.teeth("L%d FFN-up: hi half only" % l, t["L_FFN"], mut_hi)
    # FFN-down + LN (norm3 in the decoders, norm2 in the encoder)
    nn, swap = ("norm3", "norm2") if c.dec else ("norm2", "norm1")
    w2 = W("linear2.weight", kw)
    rec.same("L%d FFN-down + LN" % l, t["L_LN3"],
             resid_ln(t["L_FFN"], w2, V("linear2.bias"), V(nn + ".weight"), V(nn + ".bias"), h_ffn))
    rec.teeth("L%d FFN-down: weights of layer %d" % (l, other), t["L_LN3"],
              resid_ln(t["L_FFN"], W("linear2.weight", kw, other), V("linear2.bias", other), V(nn + ".weight", other),
                       V(nn + ".bias", other), h_ffn))
    rec.teeth("L%d FFN-down: %s for %s" % (l, swap, nn), t["L_LN3"],
              resid_ln(t["L_FFN"], w2, V("linear2.bias"), V(swap + ".weight"), V(swap + ".bias"), h_ffn))
    if c.dip:
        rec.teeth("L%d FFN-down: hi half only" % l, t["L_LN3"],
                  resid_ln(t["L_FFN"][:, :FF].contiguous(), W("linear2.weight"), V("linear2.bias"), V(nn + ".weight"),
                           V(nn + ".bias"), h_ffn))
    if l == c.L - 1:
        check_output(c, t, out, rec)


def check_output(c, t, out, rec):
    """The CFG blend (restated in torch fp32, the kernel's operation order) and the output GEMM's hook."""
    B, T, S, d = c.B, c.T, c.S, D
    h = t["L_LN3"].view(c.halves, B, S, 2 * d)[:, :, c.s_off:]
    a = h[0, ..., :d].float() + h[0, ..., d:].float()
    if c.halves == 2:
        u = h[1, ..., :d].float() + h[1, ..., d:].float()
        a = u + c.scale.view(B, 1, 1) * (a - u)
    hi = a.half()
    rec.same("CFG blend", t["BLEND"], torch.cat([hi, (a - hi.float()).half(), hi], -1).reshape(B * T, 3 * d))
    x = c.x.reshape(B, c.JF, T).contiguous()
    w_out, b_out = c.W["output_process.poseFinal.weight"], c.W["output_process.poseFinal.bias"]
    rec.same("output GEMM", out.reshape(B, c.JF, T), out_x0(t["L_LN3"], c.scale, w_out, b_out, x, c.s_off, c.halves))
    if c.halves == 2:   # the scale applied to the unconditional half: the halves swapped
        sw = t["L_LN3"].view(2, -1, 2 * d).flip(0).reshape(-1, 2 * d).contiguous()
        rec.teeth("output: scale on the unconditional half", out.reshape(B, c.JF, T),
                  out_x0(sw, c.scale, w_out, b_out, x, c.s_off, c.halves))
    else:
        rec.teeth("output: residual before the last FFN", out.reshape(B, c.JF, T),
                  out_x0(t["L_LN1"], c.scale, w_out, b_out, x, c.s_off, c.halves))


def check_entry(c, t, rec):
    """Embedding, token 0 / memory build, the all-layer K/V GEMM, and the layer-0 entry."""
    B, T, S, d = c.B, c.T, c.S, D
    w_in, b_in = c.W["input_process.poseEmbedding.weight"], c.W["input_process.poseEmbedding.bias"]
    x = c.x.reshape(B, c.JF, T)
    s_off = 1
    if c.dip:   # the prefix frames precede x: one embedding over ctx + T frames, s_off 0
        x = torch.cat([c.y["prefix"].reshape(B, c.JF, c.ctx), x], -1) if c.ctx else x
        s_off = 0
    x = x.contiguous()
    rec.same("embedding GEMM", t["EMBED"], embed(x, w_in, b_in, c.pe, s_off, c.halves))
    rec.teeth("embedding: pe shifted by one row", t["EMBED"], embed(x, w_in, b_in, c.pe[1:].contiguous(), s_off, c.halves))
    if c.dip:
        rec.same("token rows untouched by the memory build", t["TOK0"], t["EMBED"])
        wkv = torch.cat([lw(c, l, "multihead_attn.in_proj_weight")[d:] for l in range(c.L)])
        bkv = torch.cat([lw(c, l, "multihead_attn.in_proj_bias")[d:] for l in range(c.L)])
        a = t["MEM16"][:, :d].contiguous()
        rec.same("all-layer K/V GEMM", t["KVC16"], gemm_epi(a, f16(wkv), bkv, 1))
        if c.L > 1:
            wr = torch.cat([lw(c, l, "multihead_attn.in_proj_weight")[d:] for l in reversed(range(c.L))])
            br = torch.cat([lw(c, l, "multihead_attn.in_proj_bias")[d:] for l in reversed(range(c.L))])
            rec.teeth("K/V: layers in reverse order", t["KVC16"], gemm_epi(a, f16(wr), br, 1))
    else:
        # token 0, bit-exact in fp32 in the kernel's order: (condproj + (temb + g)) + pe[0]; no text term in the decoder
        hs = t["TOK0"].view(c.Bp, S, 2 * d)
        es = t["EMBED"].view(c.Bp, S, 2 * d)
        rec.same("frame rows untouched by token 0", hs[:, 1:], es[:, 1:])
        te = t["TEMB"].repeat(c.halves, 1)
        if c.g is not None:
            te = te + c.g.repeat(c.halves, 1)
        pe0 = c.pe[0]
        v = te + pe0 if c.dec else (t["CONDPROJ"] + te) + pe0
        hi = v.half()
        rec.same("token-0 row (fp32 restatement)", hs[:, 0], torch.cat([hi, (v - hi.float()).half()], -1))
        mut = te + (c.pe[1]) if c.dec else t["CONDPROJ"] + (te + pe0)
        hm = mut.half()
        rec.teeth("token 0: %s" % ("pe[1]" if c.dec else "condproj + (temb + pe[0])"), hs[:, 0],
                  torch.cat([hm, (mut - hm.float()).half()], -1))
    rec.same("layer-0 entry", t["L_IN"], t["TOK0"])


# ------------------------------------------------------------------------------------------------ (c): fp64
def linear_bound(x, w, b):
    """small_linear_kernel's error on x @ w.T + b (fp64 operands): each lane a fmaf chain of K/32 terms, a 5-level
    shuffle tree, then the bias: gamma_{K/32 + 6} (|x| |w|^T + |b|)."""
    n = -(-x.shape[-1] // 32) + 6
    g = n * U32 / (1 - n * U32)
    return g * (x.abs() @ w.abs().t() + (b.abs() if b is not None else 0))


def temb64(c, t):
    """fp64 timestep embedding of model timesteps t [n] and its bound: Linear -> SiLU -> Linear on pe[t]; the SiLU
    z / (1 + expf(-z)) adds expf's 2 ulp, the add and the division (8 u relative, with slack)."""
    W = {k: c.W["embed_timestep.time_embed.%s" % k].double() for k in ("0.weight", "0.bias", "2.weight", "2.bias")}
    p = c.pe[t].double()
    z = p @ W["0.weight"].t() + W["0.bias"]
    bz = linear_bound(p, W["0.weight"], W["0.bias"])
    s = z * torch.sigmoid(z)
    bs = 1.1 * bz + 8 * U32 * (s.abs() + 1.1 * bz)
    out = s @ W["2.weight"].t() + W["2.bias"]
    bound = bs @ W["2.weight"].abs().t() + linear_bound(s.abs() + bs, W["2.weight"], W["2.bias"])
    nosilu = z @ W["2.weight"].t() + W["2.bias"]
    return out, bound, nosilu


def check_fp64(c, t, rec):
    B, d, ts = c.B, D, c.ts.cuda()
    ref, bound, nosilu = temb64(c, ts)
    got = t["TEMB"].double()
    ref1 = temb64(c, ts + 1)[0]
    rec.bound("timestep-embedding rows", (got - ref).abs(), bound,
              {"row t + 1": (got - ref1).abs(), "SiLU dropped": (got - nosilu).abs()})
    if c.kind in ("enc", "dec_emb"):
        te = c.y["text_embed"].reshape(B, -1).double()
        w, b = c.W["embed_text.weight"].double(), c.W["embed_text.bias"].double()
        cp = t["CONDPROJ"].double()
        want = te @ w.t() + b
        mutants = {"bias dropped": (cp[:B] - want + b).abs()}
        if B > 1:
            mutants["text of sample b + 1"] = (cp[:B] - want.roll(1, 0)).abs()
        rec.bound("conditioning rows (text projection)", (cp[:B] - want).abs(), linear_bound(te, w, b), mutants)
        if c.halves == 2:
            rec.same("unconditional rows = embed_text.bias", t["CONDPROJ"][B:], c.W["embed_text.bias"].expand(B, d))
    elif c.kind == "a2m":
        act = c.W["embed_action.action_embedding"][c.y["action"].reshape(-1)]
        rec.same("conditioning rows = action embedding", t["CONDPROJ"][:B], act)
        rec.teeth("action rows: action + 1", t["CONDPROJ"][:B],
                  c.W["embed_action.action_embedding"][(c.y["action"].reshape(-1) + 1) % 12])
    if c.dip:
        Mt, H = c.Mt, c.halves
        enc = c.y["text_embed"][0].permute(1, 0, 2).double()           # [B, Mt, 768]
        w, b = c.W["embed_text.weight"].double(), c.W["embed_text.bias"].double()
        proj = enc @ w.t() + b
        pbound = linear_bound(enc, w, b)
        if H == 2:
            proj = torch.cat([proj, b.expand(B, Mt, d)])
            pbound = torch.cat([pbound, torch.zeros_like(pbound)])
        tt = ref.repeat(H, 1)[:, None]
        want = proj + tt
        m = t["MEM16"].view(H * B, Mt, 2 * d)
        got = m[..., :d].double() + m[..., d:].double()
        bnd = pbound + bound.repeat(H, 1)[:, None] + U32 * want.abs() + 2.0 ** -22 * want.abs() + 2.0 ** -25
        shifted = ref.roll(1, 0).repeat(H, 1)
        if H == 2:   # the unconditional half with the timestep of another sample (b' rather than b' mod B)
            shifted[:B] = ref
        rec.bound("DiP memory rows (text + temb)", (got - want).abs(), bnd,
                  {"timestep of another sample": (got - proj - shifted[:, None]).abs(),
                   "text bias dropped": (got - want + b).abs()})


# ------------------------------------------------------------------------------------------------ drivers
def run_case(c, title, layers=None):
    rec = Record(title)
    outs = []
    for l in (layers if layers is not None else sorted({0, c.L - 1})):
        out, t = c.eng.forward_taps(c.x, c.ts, l)
        torch.cuda.synchronize()
        if l == 0:
            check_entry(c, t, rec)
            check_fp64(c, t, rec)
        check_layer(c, l, t, out, rec)
        outs.append(out)
    plain = c.eng.denoise(c.x, c.ts)
    for o in outs:
        rec.same("tapped forward = b200mdm_denoise", o, plain)
    rec.done()


def _lengths(B, T, seed):
    ln = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed))
    ln[0] = T
    if B > 1:
        ln[1] = 1
    return ln.tolist()


def test_stages_trans_enc_text_cfg_b64():
    """The headline shape: B = 64, T = 196, L = 8, guidance scales 0 / 1 / 2.5 / 7.5, lengths including 1 and T."""
    B, T = 64, 196
    scale = torch.tensor([0.0, 1.0, 2.5, 7.5]).repeat(B // 4)
    c = build("enc", B, T, 8, 101, True, lengths=_lengths(B, T, 1), scale=scale)
    run_case(c, "trans_enc text, CFG, B=64 T=196 L=8")


def test_stages_kit_cfg():
    """KIT's 251 features (five zero pad columns of the input projection, no K tail, the partial output chunk at
    [224, 256)): B = 4, T = 196, L = 2, guidance 0 / 1 / 2.5 / 7.5, lengths including 1; then a 3-step loop against the fp32
    oracle."""
    B, T = 4, 196
    c = build("enc", B, T, 2, 191, True, lengths=[196, 1, 120, 57], scale=torch.tensor([0.0, 1.0, 2.5, 7.5]), dataset="kit")
    assert c.JF == 251 and c.eng.cfg.njoints * c.eng.cfg.nfeats == 251
    run_case(c, "KIT (251 features), CFG, B=4 T=196 L=2")
    c.inp["scale"] = torch.tensor([0.0, 1.0, 2.5, 2.5])   # (7.5 on trans_enc: the open xfail of test_precision_margin_gpu.py)
    c.y["scale"] = c.inp["scale"].cuda()
    _loop_vs_oracle(c)


def test_stages_dip_kit():
    """DiP (BERT, ctx 20 + pred 40) at KIT's 251 features: the prefix, packed by b200mdm_set_prefix at row 0 of each
    sequence and the frames at row 20, then a 3-step loop against the fp32 oracle."""
    c = build("dip", 3, 40, 2, 197, True, lengths=[40, 1, 27], scale=torch.tensor([7.5, 2.5, 1.0]), Mt=16, dataset="kit")
    assert c.JF == 251 and tuple(c.y["prefix"].shape) == (3, 251, 1, 20)
    run_case(c, "DiP ctx 20 + 40 at 251 features, CFG, B=3 L=2")
    _loop_vs_oracle(c)


def test_stages_trans_enc_target():
    c = build("enc", 4, 24, 2, 111, True, lengths=[24, 1, 11, 6], scale=torch.tensor([2.5, 1.0, 7.5, 0.0]),
              target="single")
    run_case(c, "trans_enc text + target, CFG, B=4 T=24 L=2")


def test_stages_a2m_unguided():
    c = build("a2m", 8, 60, 2, 121, False, lengths=_lengths(8, 60, 2))
    run_case(c, "a2m, B=8 T=60 L=2")


@pytest.mark.parametrize("Mt", [16, 150])
def test_stages_dip(Mt):
    """ctx 20 + pred 40; Mt = 16 (ragged mask, the register-resident core) and 150 (the key-blocked core)."""
    c = build("dip", 3, 40, 2, 131 + Mt, True, lengths=[40, 1, 27], scale=torch.tensor([7.5, 2.5, 1.0]), Mt=Mt)
    run_case(c, "DiP ctx 20 + 40, Mt=%d, CFG, B=3 L=2" % Mt)


def test_stages_bert_decoder_ctx0():
    c = build("dip", 2, 196, 2, 141, True, lengths=[196, 1], scale=torch.tensor([2.5, 7.5]), Mt=100, ctx=0)
    run_case(c, "BERT decoder, ctx 0, T=196 Mt=100, CFG, B=2 L=2")


def test_stages_clip_decoder():
    c = build("dec_emb", 3, 196, 2, 151, True, lengths=[196, 1, 80], scale=torch.tensor([7.5, 2.5, 0.0]))
    run_case(c, "CLIP decoder, T=196, CFG, B=3 L=2")


# ------------------------------------------------------------------------------------------------ shape envelope
def _loop_vs_oracle(c):
    """A 3-step DDPM loop through the engine against the fp32 oracle, per sample at 1e-3."""
    from oracle import mdm_oracle as mo, schedule_oracle as so
    from precision_cases import rel_err_per_sample
    steps = 3
    diffusion = b200mdm.create_model_and_diffusion(default_args(layers=c.L, diffusion_steps=steps),
                                                   SimpleNamespace(dataset=SimpleNamespace()))[1]
    tape = [v.cuda() for v in c.inp["tape"]]
    net = b200mdm.ClassifierFreeSampleModel(c.model)
    got = diffusion.p_sample_loop(net, c.shape, noise=tape[0], clip_denoised=False, model_kwargs={"y": c.y},
                                  noise_tape=torch.stack(tape[1:])).cpu()
    W = mo.OracleWeights(c.sd, c.L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    cpu_tape = [v.cpu() for v in c.inp["tape"]]
    sc, ln = c.inp["scale"], c.inp["lengths"]
    if c.dip:
        enc, tmask = c.y["text_embed"]
        want = mo.sample_loop_dec(W, tabs, list(range(steps)), cpu_tape, enc.cpu(), tmask.cpu(), c.y["prefix"].cpu(), sc, ln)
    else:
        want = mo.sample_loop(W, tabs, list(range(steps)), cpu_tape, c.inp["text_embed"], sc, ln)
    e = rel_err_per_sample(got, want)
    print("  3-step loop vs fp32 oracle, per sample: %s" % " ".join("%.2e" % v for v in e.tolist()))
    assert (e < 1e-3).all()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [63, 64, 207, 208, 255])
def test_shape_envelope_trans_enc(T, B):
    """S = 64 / 65 / 208 / 209 / 256: both sides of the attention core's two key-width switches, and its largest.
    Guidance stays at or below 2.5 here: the trans_enc model at 7.5 is the open precision xfail of
    test_precision_margin_gpu.py (about 1.1e-3 per sample after this loop, on its length-1 sample)."""
    lengths = [T - 1] if B == 1 else [T, 1, max(1, T // 3)]   # (one padded key at B = 1: kvlen + 1 must differ)
    scale = torch.tensor([2.5] if B == 1 else [2.5, 1.0, 0.0])
    c = build("enc", B, T, 2, 161 + T, True, lengths=lengths, scale=scale)
    run_case(c, "trans_enc text, CFG, B=%d T=%d (S=%d) L=2" % (B, T, T + 1))
    _loop_vs_oracle(c)


def test_shape_envelope_dip_s256():
    c = build("dip", 2, 236, 2, 171, True, lengths=[236, 100], scale=torch.tensor([7.5, 2.5]), Mt=16)
    run_case(c, "DiP ctx 20 + 236 (S=256), Mt=16, CFG, B=2 L=2")
    _loop_vs_oracle(c)


def test_sequences_past_256_tokens_are_refused():
    from b200mdm import _lib as L
    c = build("enc", 1, 24, 1, 181, True)
    y = dict(c.y, mask=torch.ones(1, 1, 1, 256, dtype=torch.bool, device="cuda"), lengths=torch.tensor([256], device="cuda"))
    with pytest.raises(L.B200MDMError) as ei:
        c.eng.set_cond(1, 256, y, True, "cuda")
    assert ei.value.code == L.ENOTIMPL
    d = build("dip", 1, 40, 1, 182, True, Mt=8)
    y = dict(d.y, mask=torch.ones(1, 1, 1, 237, dtype=torch.bool, device="cuda"), lengths=torch.tensor([237], device="cuda"))
    with pytest.raises(L.B200MDMError) as ei:
        d.eng.set_cond(1, 237, y, True, "cuda")
    assert ei.value.code == L.ENOTIMPL


# ------------------------------------------------------------------------------------------------ PDL off = on
PDL_KINDS = {
    "enc": lambda: build("enc", 4, 40, 2, 191, True, lengths=[40, 1, 17, 33], scale=torch.tensor([2.5, 7.5, 1.0, 0.0])),
    "a2m": lambda: build("a2m", 3, 60, 2, 192, False, lengths=[60, 1, 31]),
    "dip": lambda: build("dip", 3, 40, 2, 193, True, lengths=[40, 1, 27], scale=torch.tensor([7.5, 2.5, 1.0]), Mt=16),
    "dec_emb": lambda: build("dec_emb", 3, 40, 2, 194, True, lengths=[40, 1, 17], scale=torch.tensor([7.5, 2.5, 0.0])),
}


def pdl_loops():
    """{kind/graph|eager: 3-step DDIM loop result} for the four model kinds."""
    res = {}
    for kind, make in PDL_KINDS.items():
        c = make()
        steps = 3
        diffusion = b200mdm.create_model_and_diffusion(default_args(layers=c.L, diffusion_steps=steps),
                                                       SimpleNamespace(dataset=SimpleNamespace()))[1]
        net = b200mdm.ClassifierFreeSampleModel(c.model) if c.guided else c.model
        tape = [v.cuda() for v in c.inp["tape"]]
        for name, graph in (("graph", True), ("eager", False)):
            res["%s/%s" % (kind, name)] = diffusion.ddim_sample_loop(
                net, c.shape, noise=tape[0], clip_denoised=False, eta=0.0, model_kwargs={"y": c.y},
                noise_tape=torch.stack(tape[1:]), use_graph=graph).cpu()
    return res


def test_pdl_off_equals_pdl_on():
    """A kernel that read its predecessor's output before griddepcontrol.wait would make the result depend on timing:
    the same loops with plain stream order (B200MDM_PDL=0, a child process) must give the same bits."""
    on = pdl_loops()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pdl_off.pt")
        env = dict(os.environ, B200MDM_PDL="0")
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
        proc = subprocess.run(cmd, env=env, cwd=os.path.dirname(HERE), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True, timeout=900)
        assert proc.returncode == 0, proc.stdout[-4000:]
        off = torch.load(path)
    assert set(off) == set(on)
    bad = []
    for k in sorted(on):
        n = int((on[k].view(torch.int32) != off[k].view(torch.int32)).sum())
        print("  %-16s PDL off vs on: %d differing elements" % (k, n))
        if n:
            bad.append(k)
    assert not bad, bad


if __name__ == "__main__":
    assert os.environ.get("B200MDM_PDL") == "0"
    torch.save(pdl_loops(), sys.argv[1])
