"""GPU: each hand-written kernel against a plain torch fp32 restatement of the same op (through the C ABI)."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from b200mdm import _lib as L
    return L, L.load()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("M,N,K,bn,act", [
    (128, 256, 64, 128, 0),          # two N tiles, one k-block
    (128, 256, 512, 128, 0),         # k pipeline wraps the ring
    (300, 512, 512, 128, 0),         # M tail (300 = 2*128 + 44), 4 N tiles
    (25216 // 8, 1536, 512, 128, 0),  # QKV shape (M scaled down), many tiles per CTA
    (1000, 1024, 512, 128, 1),       # FFN up + exact GELU
    (777, 512, 1024, 128, 0),        # FFN down shape
    (394, 512, 792, 128, 0),         # embed GEMM: K = 3*264 (K tail: 792 = 12*64 + 24), BLOCK_N 128
    (394, 288, 1536, 128, 0),        # N tail inside a 128-wide tile, 64-column slab clipped by the TMA store
    (394, 264, 1536, 128, 0),        # N tail that ends inside a 32-column chunk
    (5, 16, 8, 128, 1),              # tiny
    (256, 256, 64, 512, 0),          # 128 x 256 tiles: two row tiles, one k-block
    (700, 512, 512, 512, 0),         # 256-wide: M tail inside the second warpgroup's rows (700 = 5*128 + 60), pipeline wraps
    (25216 // 8, 1536, 512, 512, 0), # 256-wide: QKV shape
    (3000, 1024, 512, 512, 1),       # 256-wide: FFN up + GELU, two staging rounds per tile
    (130, 512, 1024, 512, 0),        # 256-wide: last row tile holds 2 live rows only
    (100, 264, 512, 512, 0),         # 256-wide: second warpgroup entirely out of range, N tail in the second tile
    (256, 256, 64, 513, 0),          # W-resident kernel (128 x 64 tiles): one resident k-block
    (700, 512, 512, 513, 0),         # W-resident: M tail, one row tile per CTA
    (25216 // 8, 1536, 512, 513, 0), # W-resident: QKV shape, 24 column blocks
    (25216, 1024, 512, 513, 1),      # W-resident: the FFN up-projection at BASELINE config 2 (the A ring wraps for many
                                     # rounds while W stays put) + GELU
    (40000, 512, 320, 513, 0),       # W-resident: 5 k-blocks, many rounds
    (5000, 768, 200, 513, 1),        # W-resident: K tail inside the last k-block (200 = 3*64 + 8)
    (100, 264, 512, 513, 0),         # W-resident: second warpgroup entirely out of range, N tail
])
def test_gemm_tcgen05(M, N, K, bn, act):
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, device="cuda", generator=g)).half()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_gemm_f16(_p(a), _p(w), _p(bias), _p(out), M, N, K, act, bn, _stream()))
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias
    if act:
        ref = torch.nn.functional.gelu(ref)
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out.float()).all()
    assert err < 4e-3 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("n,S,Mt,ld_extra", [(5, 60, 16, 0), (3, 60, 16, 7168), (2, 17, 5, 0), (3, 100, 24, 0), (2, 64, 33, 1024),
                                             (2, 61, 64, 0), (1, 1, 1, 0)])
def test_cross_attention(n, S, Mt, ld_extra):
    """The trans_dec cross-attention core (mma.sync tiles, P = hi + lo) against torch fp32: padding masks, token counts
    that do not fill a key tile, rows that do not fill a 16-row tile, k | v embedded in a wider row (all-layer projection)."""
    L, lib = _lib()
    d, H, dh = 512, 4, 128
    g = torch.Generator(device="cuda").manual_seed(100 * S + Mt)
    q = torch.randn(n * S, d, device="cuda", generator=g).half()
    ld = 2 * d + ld_extra
    kvw = torch.randn(n * Mt, ld, device="cuda", generator=g).half()
    col0 = ld_extra // 2 if ld_extra else 0                          # this "layer"'s k | v columns inside the wide row
    col0 -= col0 % 8
    mask = torch.rand(n, Mt, device="cuda", generator=g) < 0.3
    mask[:, 0] = False                                               # the CLS token is never padding
    out = torch.full((n * S, 2 * d), float("nan"), device="cuda", dtype=torch.float16)
    kv_ptr = kvw.data_ptr() + 2 * col0
    L.check(lib.b200mdm_test_cross_attention(_p(q), ctypes.c_void_p(kv_ptr), _p(mask.to(torch.uint8)), _p(out), n, S, Mt, ld,
                                             _stream()))
    torch.cuda.synchronize()
    k = kvw[:, col0:col0 + d].float().view(n, Mt, H, dh).permute(0, 2, 1, 3)
    v = kvw[:, col0 + d:col0 + 2 * d].float().view(n, Mt, H, dh).permute(0, 2, 1, 3)
    qq = q.float().view(n, S, H, dh).permute(0, 2, 1, 3)
    s = qq @ k.transpose(-1, -2) / dh ** 0.5
    s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(n * S, d)
    got = out[:, :d].float()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    assert err < 1.5e-3 * max(1.0, ref.abs().max().item()), err      # fp16 output rounding (2^-11 relative) dominates


@pytest.mark.parametrize("impl", [0])
@pytest.mark.parametrize("n,S,kv", [(3, 197, [197, 121, 58]), (2, 41, [41, 1]), (4, 61, [61, 46, 31, 2]), (1, 16, [16]),
                                    (2, 33, [20, 33]), (2, 256, [256, 130]), (2, 129, [129, 128])])
def test_attention(n, S, kv, impl):
    L, lib = _lib()
    d, H, dh = 512, 4, 128
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv = torch.randn(n * S, 3 * d, device="cuda", generator=g).half()
    kvlen = torch.tensor(kv, device="cuda", dtype=torch.int32)
    out = torch.full((n * S, d), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_attention(_p(qkv), _p(out), _p(kvlen), n, S, d, impl, _stream()))
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(n, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / dh ** 0.5
    mask = torch.arange(S, device="cuda")[None, :] >= kvlen[:, None]
    s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(n * S, d)
    assert torch.isfinite(out.float()).all()
    assert (out.float() - ref).abs().max().item() < 5e-3


def _half_ulp16(v):
    """Half the fp16 spacing at |v| (the larger spacing at a binade edge)."""
    h = v.abs().float().clamp(max=65504.0).half().double()
    _, e = torch.frexp(h)
    e = torch.where(h == 0, torch.full_like(e, -13), e)
    return torch.ldexp(torch.ones_like(h), (e - 1).clamp(min=-14) - 11)


def _attn_emulate(s, v, valid, max_keys, c):
    """fp64 restatement of attention_tc_kernel for exact fp32 logits s [n, H, S, S] (raw q.k) and v [n, H, S, dh]:
    offset m = fp32(max over `max_keys` of s * c), p = 2^fp32(s c - m) (fmaf: one rounding), P = fp16(p) in P V, the row
    sum of the unrounded p.  Returns O, A = sum P |v| / l (the magnitude the accumulation works at) and F = sum over the
    keys whose p lies within the ex2.approx error (2^-21 relative) of an fp16 rounding boundary of ulp16(p) |v| / l
    (those may round either way)."""
    m = s.masked_fill(~max_keys, float("-inf")).amax(-1, keepdim=True)
    off = (m * c).float().double()
    p = torch.exp2((s * c - off).float().double()).masked_fill(~valid, 0.0)
    P = p.float().half().double()
    l = p.sum(-1, keepdim=True)
    d = 2.0 ** -21
    flip = (p * (1 + d)).float().half() != (p * (1 - d)).float().half()
    U = torch.where(flip, 2 * _half_ulp16(p), torch.zeros_like(p))
    va = v.abs()
    return (P @ v) / l, (P @ va) / l, (U @ va) / l


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("n,S,kv", [(4, 60, [60, 1, 16, 17]), (5, 197, [197, 1, 16, 17, 150]), (3, 209, [209, 17, 200]),
                                    (4, 256, [256, 1, 16, 129]), (256, 60, "mixed")])
def test_attention_peaked(n, S, kv, impl):
    """Both attention_tc_kernel variants (impl 0: fp16 out, the encoder; impl 1: [hi | lo] out, DiP) on peaked softmax
    rows, against an fp64 restatement of the kernel's arithmetic.  q = integers in [-6, 6], k = halves in [-3, 3]: every
    logit is exact in fp32, so the only differences are ex2.approx, the fp32 row sum and P V accumulation, and the output
    rounding.  Logits span about +-30 / sqrt(128)-scaled; the first masked key of every sample (key kvlen) carries the
    row's largest logit (~100), so a kernel that lets a masked key into the maximum or the sum fails.  S = 209 is above
    the 208 keys two CTAs per SM hold; S > 128 has a second query tile."""
    L, lib = _lib()
    d, H, dh = 512, 4, 128
    if kv == "mixed":
        kv = [[60, 1, 16, 17, 33, 59][i % 6] for i in range(n)]
    g = torch.Generator(device="cuda").manual_seed(S * 31 + n)
    sign = torch.randint(0, 2, (n, 1, H, dh), device="cuda", generator=g).float() * 2 - 1
    q = sign * torch.randint(0, 7, (n, S, H, dh), device="cuda", generator=g).float()
    k = torch.randint(-6, 7, (n, S, H, dh), device="cuda", generator=g).float() / 2
    kvlen = torch.tensor(kv, device="cuda", dtype=torch.int32)
    for i, kl in enumerate(kv):
        if kl < S:
            k[i, kl] = 3 * sign[i, 0]                          # aligned with every query row of the sample: the largest logit
    v = torch.randn(n, S, H, dh, device="cuda", generator=g)
    qkv = torch.cat([q.reshape(n * S, d), k.reshape(n * S, d), v.reshape(n * S, d)], 1).half().contiguous()
    out = torch.full((n * S, (2 if impl else 1) * d), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_attention(_p(qkv), _p(out), _p(kvlen), n, S, d, impl, _stream()))
    torch.cuda.synchronize()

    qq, kk, vv = (t.double().permute(0, 2, 1, 3) for t in (q, k, qkv[:, 2 * d:].view(n, S, H, dh)))
    s = qq @ kk.transpose(-1, -2)                              # exact: multiples of 1/2 below 2^12
    c = float(np.float32(np.float32(1.4426950408889634) / np.sqrt(np.float32(128.0))))
    key = torch.arange(S, device="cuda")
    valid = (key[None, :] < kvlen[:, None])[:, None, None, :]
    O, A, F = _attn_emulate(s, vv, valid, valid, c)
    blocks = ((kvlen.clamp(max=S) + 15) // 16).double()[:, None, None, None]
    # P V over 16*blocks keys (accumulator updates every ACC_CHUNK = 4 products, 2^-23 each, of a partial sum <= A l);
    # row sum: 4 fp32 adds per block + 2 shuffles; ex2.approx 2^-21 on l; 1/l, O * (1/l) and hi + lo: 4 roundings
    rel = 4 * blocks * 2.0 ** -23 + (4 * blocks + 2) * 2.0 ** -24 + 2.0 ** -21 + 4 * 2.0 ** -24
    slack = rel * A + F
    mx = _attn_emulate(s, vv, valid, (key < S)[None, None, None, :].expand_as(valid), c)[0]
    plus1 = (key[None, :] < (kvlen.clamp(max=S - 1) + 1)[:, None])[:, None, None, :]
    k1 = _attn_emulate(s, vv, plus1, plus1, c)[0]

    def rows(t):                                               # [n, H, S, dh] -> [n*S, d]
        return t.permute(0, 2, 1, 3).reshape(n * S, d)
    O, slack, mx, k1 = rows(O), rows(slack), rows(mx), rows(k1)
    if impl == 0:
        got = out.double()
        bound = _half_ulp16(O.abs() + slack) + slack
        mutants = {"max over all keys": (mx.float().half().double() - O).abs(),
                   "kvlen + 1 keys": (k1.float().half().double() - O).abs()}
    else:
        hi = out[:, :d].double()
        got = hi + out[:, d:].double()
        bound = slack + 2.0 ** -22 * O.abs() + 2.0 ** -25
        mutants = {"max over all keys": (mx - O).abs(), "kvlen + 1 keys": (k1 - O).abs(), "lo half zeroed": (hi - O).abs()}
    err = (got - O).abs()
    ratio = (err / bound).max().item()
    msg = ["attention impl=%d n=%d S=%d: kernel error / bound = %.3g" % (impl, n, S, ratio)]
    bad = []
    for name, me in mutants.items():
        mr = (me / bound).max().item()
        msg.append("  mutant %-20s error / bound = %.3g" % (name + ":", mr))
        if not mr >= 8:
            bad.append(name)
    print("\n".join(msg))
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, ratio
    assert not bad, bad


@pytest.mark.parametrize("n,S,kv,ld", [(3, 197, [197, 121, 58], 1024), (2, 41, [41, 1], 512), (4, 61, [61, 46, 31, 2], 512),
                                       (1, 16, [16], 512), (2, 256, [256, 130], 1024), (2, 129, [129, 128], 512),
                                       (2, 128, [128, 7], 512), (40, 197, [197] * 39 + [3], 1024)])
def test_qkv_attention_fused(n, S, kv, ld):
    """QKV projection + attention core of an encoder layer (the QKV GEMM and the attention kernel the step launches) vs
    torch fp32 on the same fp16 operands; `ld` = 1024 feeds it the hi half of an [hi | lo] residual stream like the engine
    does; 40 samples exercise many row tiles per CTA of the GEMM and 320 CTAs of the attention kernel."""
    L, lib = _lib()
    d, H, dh = 512, 4, 128
    g = torch.Generator(device="cuda").manual_seed(S * 7 + n)
    h = torch.randn(n * S, ld, device="cuda", generator=g).half()
    w = (torch.randn(3 * d, d, device="cuda", generator=g) / d ** 0.5).half()
    bias = torch.randn(3 * d, device="cuda", generator=g) * 0.3
    kvlen = torch.tensor(kv, device="cuda", dtype=torch.int32)
    out = torch.full((n * S, d), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_qkv_attention(_p(h), ld, _p(w), _p(bias), _p(out), _p(kvlen), n, S, _stream()))
    torch.cuda.synchronize()
    qkv = (h[:, :d].float() @ w.float().t() + bias).half().float()           # the kernel keeps q, k, v in fp16
    q, k, v = qkv.view(n, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    s_ = q @ k.transpose(-1, -2) / dh ** 0.5
    mask = torch.arange(S, device="cuda")[None, :] >= kvlen[:, None]
    s_ = s_.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s_, -1) @ v).permute(0, 2, 1, 3).reshape(n * S, d)
    assert torch.isfinite(out.float()).all()
    err = (out.float() - ref).abs().max().item()
    assert err < 5e-3, err


def _split_hi_lo(x):
    hi = x.half()
    return torch.cat([hi, (x - hi.float()).half()], dim=1).contiguous()


@pytest.mark.parametrize("M,K", [(256, 512), (25216 // 4, 512), (3000, 1024), (130, 512), (77, 1024), (25216, 512), (25216, 2048)])
def test_gemm_residual_layernorm_fused(M, K):
    """h <- LN(h + A W^T + b): the fused out-projection / FFN-down kernel vs torch fp32.  h travels as the engine's
    residual-stream format, fp16 [hi | lo] (hi + lo ~ 22 bits)."""
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    w = (torch.randn(512, K, device="cuda", generator=g) / K ** 0.5).half()
    bias = torch.randn(512, device="cuda", generator=g) * 0.1
    gamma = 1 + 0.1 * torch.randn(512, device="cuda", generator=g)
    beta = 0.1 * torch.randn(512, device="cuda", generator=g)
    h = torch.randn(M, 512, device="cuda", generator=g) * 1.5 + 0.2
    hres = _split_hi_lo(h)
    h_in = hres[:, :512].float() + hres[:, 512:].float()        # what the kernel reads (|h_in - h| < 1e-6)
    ref = torch.nn.functional.layer_norm(h_in + a.float() @ w.float().t() + bias, (512,), gamma, beta, 1e-5)
    L.check(lib.b200mdm_test_gemm_resid_ln(_p(a), _p(w), _p(bias), _p(gamma), _p(beta), _p(hres), M, K, _stream()))
    torch.cuda.synchronize()
    out = hres[:, :512].float() + hres[:, 512:].float()
    assert torch.isfinite(out).all()
    assert (out - ref).abs().max().item() < 2e-4
    assert (hres[:, :512].float() - ref).abs().max().item() < 5e-3   # the hi half alone is the fp16 GEMM operand
