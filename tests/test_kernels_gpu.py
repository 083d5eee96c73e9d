"""GPU: each hand-written kernel against a plain restatement of the same op (through the C ABI): torch fp32, or fp64
with a per-element bound derived from the kernel's arithmetic and host-side mutants that must miss it (check)."""
import ctypes

import numpy as np
import pytest
import torch

from test_epilogues_gpu import (U32, acc_bound, check, gelu64, gelu_bound, gelu_tanh64, grid_operands, half_ulp16,
                                split16)

pytestmark = pytest.mark.gpu


def _lib():
    from b200mdm import _lib as L
    return L, L.load()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def run_gemm_f16(a, w, bias, act, bn):
    L, lib = _lib()
    (M, K), N = a.shape, w.shape[0]
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_gemm_f16(_p(a), _p(w), _p(bias), _p(out), M, N, K, act, bn, _stream()))
    torch.cuda.synchronize()
    return out


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
    (256, 256, 64, 128, 0),          # two row tiles, one k-block
    (256, 256, 64, 128, 1),
    (700, 512, 512, 128, 0),         # M tail of 60 rows in the last row tile (700 = 5*128 + 60), pipeline wraps
    (700, 512, 512, 128, 1),
    (25216 // 8, 1536, 512, 128, 1), # QKV shape through the GELU epilogue
    (3000, 1024, 512, 128, 1),       # FFN up + GELU, M tail of 56 rows
    (130, 512, 1024, 128, 0),        # last row tile holds 2 live rows only
    (130, 512, 1024, 128, 1),
    (100, 264, 512, 128, 0),         # one partial row tile, N tail of 8 columns in the third column tile
    (100, 264, 512, 128, 1),
    (25216, 1024, 512, 128, 1),      # the FFN up-projection at BASELINE config 2 + GELU
    (40000, 512, 320, 128, 0),       # 5 k-blocks, ten tiles per CTA
    (5000, 768, 200, 128, 1),        # K tail inside the last k-block (200 = 3*64 + 8)
])
def test_gemm_tcgen05(M, N, K, bn, act):
    """EpiBiasF16<act> behind the 128 x 128 projection GEMM (block_n = 128, the only tile shape), on grid operands (the
    fp32 accumulation is exact).  act = 0: fp16(fp32(acc + bias)) bit for bit.  act = 1: fp16(gelu_erf(fp32(acc + bias))) against fp64
    gelu(acc + bias) within half an fp16 ulp + gelu_erf's bound + the fp32 bias add (|gelu'| <= 1.13)."""
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a, w = grid_operands(M, N, K, g)
    # one bias per 12 / N stratum of [-6, 6]: every launch, down to 16 columns, crosses the whole GELU
    bias = -6 + 12 * (torch.randperm(N, device="cuda", generator=g).float() + torch.rand(N, device="cuda", generator=g)) / N
    out = run_gemm_f16(a, w, bias, act, bn)
    acc = a.double() @ w.double().t()
    if not act:
        want = (acc.float() + bias).half()
        diff = int((out.view(torch.int16) != want.view(torch.int16)).sum())
        nb16 = int(((acc.float() + bias.half().float()).half().view(torch.int16) != want.view(torch.int16)).sum())
        print("gemm f16 M=%d N=%d K=%d bn=%d: %d of %d elements differ from fp16(fp32(acc + bias)); the fp16-bias "
              "mutant differs in %d" % (M, N, K, bn, diff, want.numel(), nb16))
        assert nb16 > 0, "the bit-exact check would not see an fp16 bias"
        assert diff == 0
        return
    x = acc + bias.double()
    ref = gelu64(x)
    bound = half_ulp16(ref) + gelu_bound(ref) + 1.13 * U32 * x.abs()
    mutants = {"tanh-GELU": (gelu_tanh64(x) - ref).abs()}
    if M * N >= 4096:   # an fp16 bias shows where x is near 0 and |bias| >~ 1/4: the 80 elements of (5, 16, 8) have none
        mutants["bias rounded to fp16"] = (gelu64(acc + bias.half().double()) - ref).abs()
    if N > 32:
        mutants["bias of the next 32-column chunk"] = (gelu64(acc + bias.double().roll(-32)) - ref).abs()
    check("EpiBiasF16<GELU> M=%d N=%d K=%d bn=%d" % (M, N, K, bn), (out.double() - ref).abs(), bound, mutants)


CROSS_C = float(np.float32(np.float32(1.4426950408889634) / np.sqrt(np.float32(128.0))))   # log2(e) / sqrt(dh), fp32


def run_cross_attention(q16, kv, col0, mask, n, S, Mt):
    L, lib = _lib()
    out = torch.full((n * S, 1024), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_cross_attention(_p(q16), ctypes.c_void_p(kv.data_ptr() + 2 * col0), _p(mask.to(torch.uint8)),
                                             _p(out), n, S, Mt, kv.shape[1], _stream()))
    torch.cuda.synchronize()
    return out


def _cross_emulate(s, v, valid):
    """fp64 restatement of cross_attention_kernel for exact fp32 logits s [n, H, S, Mt] (raw q.k), v [n, H, Mt, dh] and
    the admitted keys `valid` [n, 1, 1, Mt]: sc = fp32(s c), off = max over the valid keys, p = 2^fp32(sc - off).
    Returns O = sum p v / l (l = sum p), A = sum p |v| / l and p."""
    sc = (s * CROSS_C).float()
    off = sc.masked_fill(~valid, float("-inf")).amax(-1, keepdim=True)
    p = torch.exp2((sc - off).double()).masked_fill(~valid, 0.0)
    l = p.sum(-1, keepdim=True)
    return (p @ v) / l, (p @ v.abs()) / l, p


@pytest.mark.parametrize("n,S,Mt,ld_extra", [
    (5, 60, 16, 0),             # the DiP decoder: 60 queries
    (3, 60, 16, 7168),          # k | v of layer 7 of the all-layer K/V projection row (ld_kv = 8192)
    (2, 17, 5, 0),              # tokens that do not fill a key tile, rows that do not fill a 16-row tile
    (3, 100, 24, 0),
    (2, 64, 33, 1024),
    (2, 61, 64, 0),
    (1, 1, 1, 0),
    (4, 15, 7, 0),              # MAX_NT = 2; S < 16
    (4, 65, 8, 0),              # one full key tile; a second 64-row pass of one row
    (4, 200, 17, 0),            # MAX_NT = 4 with one token in its second 16-key block; four 64-row passes
    (4, 60, 31, 0),
    (4, 17, 32, 0),             # MAX_NT = 4, full
    (4, 61, 60, 7168),          # MAX_NT = 8
    (256, 60, 64, 7168),        # the engine's launch: 2 x 128 samples, layer 7
])
def test_cross_attention(n, S, Mt, ld_extra):
    """The DiP cross-attention core (mma.sync tiles, P = hi + lo) against an fp64 restatement of its arithmetic.  k | v
    sit at the end of a row of ld_extra more columns, where the last layer's are in the all-layer K/V projection.
    q = integers in [-6, 6] (one sign per column of a sample and head), k = halves in [-3, 3]: every logit is exact in
    fp32.  Padding per sample (i mod 4): ragged, CLS only, a run in the middle, none; the first padded key of every
    sample carries the largest logit of each of its rows, and with n >= 3 the last sample is fully masked, which must
    give exactly 0.  Bound: exp2f (2 ulp) on every p, the fp16 split of P (lo rounded), the mma.sync accumulation of
    the hi and lo products (acc_bound, in the kernel's k order), the fp32 row sum of p in the kernel's order (pair
    add, chain over the key tiles, two quad shuffles), 1 / l and the product (IEEE), then half an fp16 ulp of O."""
    d, H, dh = 512, 4, 128
    ld, col0 = 2 * d + ld_extra, ld_extra
    max_nt = 2 if Mt <= 16 else 4 if Mt <= 32 else 8
    keys = 8 * max_nt
    g = torch.Generator(device="cuda").manual_seed(100 * S + Mt + n)
    sign = torch.randint(0, 2, (n, 1, H, dh), device="cuda", generator=g).float() * 2 - 1
    q = sign * torch.randint(0, 7, (n, S, H, dh), device="cuda", generator=g).float()
    k = torch.randint(-6, 7, (n, Mt, H, dh), device="cuda", generator=g).float() / 2
    mask = torch.zeros(n, Mt, dtype=torch.bool, device="cuda")
    ragged = torch.rand(n, Mt, device="cuda", generator=g) < 0.3
    for i in range(n):
        kind = i % 4
        if kind == 0:
            mask[i, 1:] = ragged[i, 1:]
        elif kind == 1:
            mask[i, 1:] = True
        elif kind == 2 and Mt >= 3:
            mask[i, Mt // 3:max(Mt // 3 + 1, 2 * Mt // 3)] = True
    full = torch.zeros(n, dtype=torch.bool, device="cuda")
    if n >= 3:
        full[-1] = True
        mask[-1] = True
    padded = mask.any(1) & ~full
    first_pad = mask.int().argmax(1)
    for i in torch.nonzero(padded).flatten().tolist():
        k[i, first_pad[i]] = 3 * sign[i, 0]                          # aligned with every query row of the sample
    kvw = torch.randn(n * Mt, ld, device="cuda", generator=g).half()
    kvw[:, col0:col0 + d] = k.reshape(n * Mt, d).half()
    q16 = q.reshape(n * S, d).half()
    out = run_cross_attention(q16, kvw, col0, mask, n, S, Mt)

    def heads(t, rows):                                               # [n * rows, d] -> [n, H, rows, dh]
        return t.double().view(n, rows, H, dh).permute(0, 2, 1, 3)
    qq, kk, vv = heads(q16, S), heads(kvw[:, col0:col0 + d], Mt), heads(kvw[:, col0 + d:col0 + 2 * d], Mt)
    got = heads(out[:, :d], S)
    assert torch.equal(got[full], torch.zeros_like(got[full])), "a fully masked row must give 0"
    s = qq @ kk.transpose(-1, -2)                                     # exact: multiples of 1/2 below 2^12
    key = torch.arange(Mt, device="cuda")
    valid = (~mask)[:, None, None, :]
    O, A, p = _cross_emulate(s, vv, valid)
    l = p.sum(-1, keepdim=True)

    # P = hi + lo: the lo rounding of p - hi (exact in fp32), p within 2^-22 of the emulated value
    pf = p.float()
    phi, plo = split16(pf)
    rem = (pf - phi.float()).double()
    e_split = torch.where(p > 0, half_ulp16(rem.abs() + 2.0 ** -22 * p), torch.zeros_like(p))
    # P V in the kernel's k order: per 16-key block, the hi products, then the lo products
    pad = keys - Mt
    P2 = torch.stack([torch.nn.functional.pad(t, (0, pad)).view(n, H, S, keys // 16, 16)
                      for t in (phi.double(), plo.double())], -2).reshape(n, H, S, 2 * keys)
    vt = torch.nn.functional.pad(vv.transpose(-1, -2), (0, pad)).view(n, H, dh, keys // 16, 16)
    V2 = torch.stack([vt, vt], -2).reshape(n, H, dh, 2 * keys)
    acc = acc_bound(P2, V2)
    # the row sum: thread t adds (p[8 nt + 2t] + p[8 nt + 2t + 1]) for nt = 0 .. MAX_NT - 1, then xor 1, xor 2
    pairs = torch.nn.functional.pad(p, (0, pad)).view(n, H, S, max_nt, 4, 2).sum(-1)
    chain = pairs.cumsum(-2)
    tot = chain[..., -1, :]
    l1 = tot.view(n, H, S, 2, 2).sum(-1)
    e_l = U32 * (pairs.sum((-1, -2)) + chain.sum((-1, -2)) + l1.sum(-1) + l[..., 0])[..., None]
    Oa = O.abs()
    dO = (2.0 ** -22 * (A + Oa) + (e_split @ vv.abs()) / l + acc / l + Oa * e_l / l + 2 * U32 * Oa) * (1 + 2.0 ** -16)
    bound = dO + half_ulp16(Oa + dO)

    def rounded(o):
        return (torch.nan_to_num(o, nan=0.0).float().half().double() - O).abs()
    O_hi = (phi.double() @ vv) / l
    admit = valid | ((key[None, :] == first_pad[:, None]) & padded[:, None])[:, None, None, :]
    last = Mt - 1 - valid[:, 0, 0].flip(-1).int().argmax(-1)
    drop = valid & (key[None, :] != last[:, None])[:, None, None, :]
    mutants = {"last valid token dropped": rounded(_cross_emulate(s, vv, drop)[0])}
    if Mt > 1:                                                        # one token: p = 1, lo = 0
        mutants["P hi only"] = rounded(O_hi)
    if padded.any():
        mutants["padded token admitted"] = rounded(_cross_emulate(s, vv, admit)[0])
    check("cross-attention n=%d S=%d Mt=%d" % (n, S, Mt), (got - O).abs(), bound, mutants, where=~full)


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
    U = torch.where(flip, 2 * half_ulp16(p), torch.zeros_like(p))
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
        bound = half_ulp16(O.abs() + slack) + slack
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


# ------------------------------------------------------------------------------------------------ residual + LayerNorm
LN_D = 512
LN_EPS = float(np.float32(1e-5))                        # GemmLnParams::eps
ORDINARY, GRID, NEAR_EPS, OFFSET = range(4)
NEAR_EPS_STEPS = [0, 30, 120, 360, 1200]                # near-eps rows: v = c0 + m 2^-16, |m| <= step (0: constant row)
OFFSET_RATIOS = [0, 8, 16, 32, 48, 64, 96, 128]         # mean-offset rows: v ~ ratio + N(0, 1)


def _ln_families(M, device):
    """Family of each row and its index in that family's parameter list: rows 8i .. 8i+3 ordinary, 8i+4 on the grid,
    8i+5 near eps, 8i+6 and 8i+7 mean-offset, so every launch mixes all four."""
    r = torch.arange(M, device=device)
    fam = torch.full((M,), ORDINARY, device=device)
    fam[r % 8 == 4] = GRID
    fam[r % 8 == 5] = NEAR_EPS
    fam[r % 8 >= 6] = OFFSET
    idx = torch.where(fam == OFFSET, 2 * (r // 8) + r % 8 - 6, r // 8)
    return fam, idx


def run_resid_ln(a, w, bias, gamma, beta, hres):
    L, lib = _lib()
    M, K = a.shape
    L.check(lib.b200mdm_test_gemm_resid_ln(_p(a), _p(w), _p(bias), _p(gamma), _p(beta), _p(hres), M, K, _stream()))
    torch.cuda.synchronize()


def _inexact(t):
    return t != t.float().double()


def _fp32_sum_error(seq, pre_inexact=None):
    """First-order bound on the rounding error of the kernel's fp32 row sum.  seq [M, 2, 4, L]: the exact (fp64) terms
    that thread t of a quad of CTA r adds into its serial chain, in order; two quad shuffles and one add of the peer
    CTA's partial then make the row sum.  Each inexact fp32 add is off by at most 2^-24 of its result (taken as the
    exact partial sum; the second-order terms are the caller's slack).  An add whose result is an fp32 value is exact
    while every operation before it was, so rows whose terms lie on a coarse grid get 0.  pre_inexact [M, 2, 4, L]:
    the terms that are themselves rounded results."""
    M = seq.shape[0]
    part = seq.cumsum(-1)
    first = _inexact(part) if pre_inexact is None else _inexact(part) | pre_inexact
    bad = torch.cummax(first.to(torch.uint8), -1)[0].bool()
    err = (part.abs() * bad).sum(-1)                                  # [M, 2, 4]
    l1 = part[..., -1].view(M, 2, 2, 2).sum(-1)                       # xor-1 shuffle
    b1 = bad[..., -1].view(M, 2, 2, 2).any(-1) | _inexact(l1)
    l2 = l1.sum(-1)                                                   # xor-2 shuffle
    b2 = b1.any(-1) | _inexact(l2)
    l3 = l2.sum(-1)                                                   # + the peer CTA's partial
    b3 = b2.any(-1) | _inexact(l3)
    return U32 * (err.sum((1, 2)) + (l1.abs() * b1).sum((1, 2)) + (l2.abs() * b2).sum(1) + l3.abs() * b3)


def ln_sum_errors(v):
    """Bounds on the errors of the kernel's two fp32 row sums of v [M, 512] (fp64, exact fp32 values).  Thread t of CTA r
    owns the column pairs (256 r + 8 j + 2 t, +1), j = 0..31: s += (v[c] + v[c+1]) rounds the pair, then the chain add
    (32 + 32 roundings); q = fmaf(v[c], v[c], fmaf(v[c+1], v[c+1], q)) adds the squares, exact inside the FMA, c+1 first
    (64 roundings)."""
    M = v.shape[0]
    x = v.view(M, 2, 32, 4, 2).permute(0, 1, 3, 2, 4)                 # [row, CTA, thread, j, pair]
    pair = x.sum(-1)
    e_s = _fp32_sum_error(pair, _inexact(pair)) + U32 * (pair.abs() * _inexact(pair)).sum((1, 2, 3))
    e_q = _fp32_sum_error((x * x).flip(-1).reshape(M, 2, 4, 64))
    return e_s, e_q


def ln_bound(v, gamma, y):
    """Per-element bound on |hi + lo - y| for the kernel's LayerNorm of the exact fp32 v [M, 512] (fp64), y the fp64
    LayerNorm of v.  Terms: the fp32 row sums (ln_sum_errors), mean = sum / 512 (exact), var = sum_sq / 512 - mean^2
    (the mean^2 product, FMA-contracted or not, and the subtraction: the one-pass cancellation term, which grows as
    (mean / std)^2), + eps, rsqrtf (2 ulp), y = ((v - mean) rstd) gamma + beta (with or without an FMA), the [hi | lo]
    split; a factor 1 + 2^-16 covers the second-order terms."""
    u, n = U32, LN_D
    e_s, e_q = ln_sum_errors(v)
    mu = v.mean(1)
    var = ((v - mu[:, None]) ** 2).mean(1)
    dmu = e_s / n
    pre = e_q / n + dmu * (2 * mu.abs() + dmu) + u * (mu.abs() + dmu) ** 2
    dvar = pre + u * (var + pre)
    w = var + LN_EPS
    dw = dvar + u * (w + dvar)
    rel_w = (dw / w).clamp(max=0.5)                   # over 0.5 the bound is void; asserted below
    assert bool((dw / w <= 0.5).all()), "LayerNorm bound: variance error over half the variance"
    R = (1 - rel_w) ** -0.5 * (1 + 2.0 ** -22) - 1    # relative error of rstd: the variance, then rsqrtf's 2 ulp
    rstd = w.rsqrt()
    R, rstd, dmu = R[:, None], rstd[:, None], dmu[:, None]
    D = (v - mu[:, None]).abs()
    dd = dmu + u * (D + dmu)                          # v - mean
    T = (D + dd) * rstd * (1 + R)
    dt = dd * rstd * (1 + R) + D * rstd * R + u * T   # (v - mean) * rstd
    G = gamma.abs()[None, :]
    dy = dt * G + u * T * G * (1 + u) + u * (y.abs() + dt * G + u * T * G)
    return (dy + 2.0 ** -22 * (y.abs() + dy) + 2.0 ** -25) * (1 + 2.0 ** -16)


def ln64(v, gamma, beta, eps=LN_EPS, n=LN_D):
    """fp64 LayerNorm over the rows of v (two-pass variance, divided by n)."""
    mu = v.mean(1, keepdim=True)
    d = v - mu
    return d / torch.sqrt((d * d).sum(1, keepdim=True) / n + eps) * gamma + beta


def ln_operands(M, K, g):
    """Inputs of one residual + LayerNorm launch.  K = 512: the encoder form, fp16 A [M, 512].  K = 1024 / 2048: the DiP
    form, A = [A_hi | A_lo] against [W | W] with A_lo = l / 1024 (|l| <= 4): products on a 2^-18 grid, partial sums
    below 2^6, so the accumulator is exact.  The bias lies on a 2^-20 grid (|b| < 1, not fp16-representable).  Rows
    other than the ordinary ones have A = 0 and a residual r = target - bias that [hi | lo] holds exactly, so the kernel
    forms v = target exactly.  Returns (a, w, bias, gamma, beta, [hi | lo] residual, target v (NaN on ordinary rows),
    A_hi W^T of the DiP form)."""
    dev = "cuda"
    fam, idx = _ln_families(M, dev)
    a, w = grid_operands(M, LN_D, K, g)
    if K > LN_D:
        a_lo = (torch.randint(-4, 5, (M, K // 2), device=dev, generator=g).float() / 1024).half()
        a = torch.cat([a[:, :K // 2], a_lo], 1)
        w = torch.cat([w[:, :K // 2], w[:, :K // 2]], 1).contiguous()
    a[fam != ORDINARY] = 0
    bias = torch.round(torch.randn(LN_D, device=dev, generator=g) * 0.1 * 2 ** 20) / 2 ** 20
    gamma = 1 + 0.1 * torch.randn(LN_D, device=dev, generator=g)
    beta = 0.1 * torch.randn(LN_D, device=dev, generator=g)

    target = torch.full((M, LN_D), float("nan"), device=dev)
    gr = fam == GRID                                                  # |v| < 4 on a 2^-5 grid: both row sums exact
    target[gr] = torch.randint(-127, 128, (int(gr.sum()), LN_D), device=dev, generator=g).float() / 32
    ne = fam == NEAR_EPS                                              # variance from 0 to about 11 eps
    step = torch.tensor(NEAR_EPS_STEPS, device=dev)[idx[ne] % len(NEAR_EPS_STEPS)]
    m = torch.round((torch.rand(int(ne.sum()), LN_D, device=dev, generator=g) * 2 - 1) * step[:, None])
    c0 = torch.randint(-64, 65, (int(ne.sum()), 1), device=dev, generator=g).float()
    c0 = torch.where(step[:, None] == 0, torch.full_like(c0, 1.5 * 2 ** 16), c0)   # the constant row: v = 1.5
    target[ne] = (c0 + m) / 2 ** 16
    h = torch.randn(M, LN_D, device=dev, generator=g) * 1.5 + 0.2   # ordinary rows
    off = fam == OFFSET
    ratio = torch.tensor(OFFSET_RATIOS, device=dev, dtype=torch.float32)[idx[off] % len(OFFSET_RATIOS)]
    h[off] = ratio[:, None] + torch.randn(int(off.sum()), LN_D, device=dev, generator=g)
    designed = gr | ne
    h[designed] = target[designed] - bias                             # exact: a multiple of 2^-20 below 2^3
    hi, lo = split16(h)
    hres = torch.cat([hi, lo], 1).contiguous()
    acc_hi = a[:, :K // 2].double() @ w[:, :K // 2].double().t() if K > LN_D else None
    return a, w, bias, gamma, beta, hres, target, acc_hi


@pytest.mark.parametrize("M,K", [
    (256, 512),
    (25216 // 4, 512), # several tiles per cluster, the last one partial
    (3000, 1024),
    (130, 512),        # two live rows in the last tile
    (77, 1024),
    (25216, 512),      # the encoder's out-proj / FFN-down at C2 (M = 2 x 64 x 197)
    (25216, 2048),
    (77, 512),         # one tile, the second warpgroup's rows wholly past M
    (300, 512),        # last tile: the second warpgroup partly live
    (15360, 1024),     # DiP out-proj: [hi | lo] attention output against [W | W] (M = 2 x 128 x 60)
    (15360, 2048),     # DiP FFN-down: [hi | lo] GELU output against [W | W]
])
def test_gemm_residual_layernorm_fused(M, K):
    """gemm_resid_ln_cluster: h <- LN(h + A W^T + b) in place on the [hi | lo] residual stream, against the fp64
    LayerNorm of the exact fp32 v = r + (acc + b) the kernel forms (r = hi + lo; the accumulator is exact), within
    ln_bound.  Four row families share each launch: ordinary rows (random residual, nonzero lo), rows on a coarse
    grid (exact row sums: the bound is tight), rows with a variance near eps (one constant row, whose output must be
    beta exactly) and mean-offset rows (mean / std up to 128), whose error against fp64 LayerNorm is printed per ratio."""
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a, w, bias, gamma, beta, hres, target, acc_hi = ln_operands(M, K, g)
    hi, lo = hres[:, :LN_D].clone(), hres[:, LN_D:].clone()
    run_resid_ln(a, w, bias, gamma, beta, hres)
    got = hres[:, :LN_D].double() + hres[:, LN_D:].double()

    fam, idx = _ln_families(M, "cuda")
    acc = (a.double() @ w.double().t()).float()                       # exact
    r = hi.float() + lo.float()
    v32 = r + (acc + bias)                                            # the kernel's v, fp32
    designed = ~torch.isnan(target[:, 0])
    assert torch.equal(v32[designed], target[designed]), "the designed rows are not exact"
    v = v32.double()
    g64, b64 = gamma.double(), beta.double()
    y = ln64(v, g64, b64)
    bound = ln_bound(v, g64, y)
    err = (got - y).abs()

    const = (fam == NEAR_EPS) & (torch.tensor(NEAR_EPS_STEPS, device="cuda")[idx % len(NEAR_EPS_STEPS)] == 0)
    bh, bl = split16(beta)
    assert torch.equal(hres[const, :LN_D].view(torch.int16), bh.expand(int(const.sum()), -1).view(torch.int16)) and \
        torch.equal(hres[const, LN_D:].view(torch.int16), bl.expand(int(const.sum()), -1).view(torch.int16)), \
        "a constant row must give beta"

    def mut(vm=None, gm=g64, bm=b64, **kw):
        return (ln64(v if vm is None else vm, gm, bm, **kw) - y).abs()
    hi_only = (y.float().half().double() - y).abs()
    var511 = mut(n=LN_D - 1)
    gb16 = mut(gm=gamma.half().double(), bm=beta.half().double())
    ordinary = {"residual lo dropped on read": mut((hi.float() + (acc + bias)).double()),
                "output lo zeroed": hi_only,
                "bias rounded to fp16": mut((r + (acc + bias.half().float())).double()),
                "gamma and beta rounded to fp16": gb16,
                "variance divided by 511": var511}
    if acc_hi is not None:
        ordinary["activation lo ignored"] = mut((r + (acc_hi.float() + bias)).double())
    name = "resid+LN M=%d K=%d" % (M, K)
    check(name + " ordinary rows", err, bound, ordinary, where=fam == ORDINARY)
    check(name + " grid rows", err, bound, {"output lo zeroed": hi_only, "gamma and beta rounded to fp16": gb16,
                                           "variance divided by 511": var511}, where=fam == GRID)
    check(name + " near-eps rows", err, bound, {"eps = 0": mut(eps=0.0)}, where=(fam == NEAR_EPS) & ~const)
    check(name + " constant rows", err, bound, {}, where=const)
    off = fam == OFFSET
    check(name + " mean-offset rows", err, bound, {}, where=off)

    # the one-pass variance on the mean-offset rows: error against fp64 LayerNorm as a fraction of max |y| of the row
    mu, sd = v.mean(1), v.std(1, unbiased=False)
    frac = err.amax(1) / y.abs().amax(1)
    line = []
    for k in range(len(OFFSET_RATIOS)):
        rows = off & (idx % len(OFFSET_RATIOS) == k)
        if rows.any():
            line.append("%.3g: %.2g" % ((mu[rows] / sd[rows]).mean().item(), frac[rows].max().item()))
    print("  mean-offset rows, mean / std: max error / max |y| --  " + ", ".join(line))
