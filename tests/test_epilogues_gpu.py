"""GPU: the split-precision GEMM epilogues of the step against fp64 references built from the exact operands the kernels
receive.  Every bound is per element and derived from the arithmetic (fp16 half-ulp, fp32 roundings, fp32 accumulation
over K, hi + lo to ~2^-22), and every bound is shown to discriminate: a plausible bug, evaluated on the host from the
same operands, must miss it by at least MUTANT_MARGIN.  Each test prints its kernel-error / bound and mutant-error /
bound ratios (the largest over all elements)."""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MUTANT_MARGIN = 8.0
U32 = 2.0 ** -24          # fp32 unit roundoff
ACC_CHUNK = 4             # products the tensor-core accumulator absorbs per update in the accumulation bound
GELU_ABS = 8e-7           # gelu_erf's documented absolute error (epilogues.cuh)
F64 = torch.float64


def _lib():
    from b200mdm import _lib as L
    return L, L.load()


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def half_ulp16(v):
    """Half the fp16 spacing at |v| (fp64 tensor).  At a binade edge |v| may round up to the power of two: the spacing
    above it, the larger one, is taken."""
    h = v.abs().float().clamp(max=65504.0).half().double()
    _, e = torch.frexp(h)
    e = torch.where(h == 0, torch.full_like(e, -13), e)
    return torch.ldexp(torch.ones_like(h), (e - 1).clamp(min=-14) - 11)


def split16(x):
    """The kernels' fp16 [hi | lo] split of fp32 x: hi = fp16(x), lo = fp16(x - hi) (x - hi is exact in fp32)."""
    hi = x.half()
    return hi, (x - hi.float()).half()


def acc_bound(a, w):
    """Bound on the fp32 accumulation error of a @ w.T on the tensor cores, from the exact operands (fp64) a [..., M, K]
    and w [..., N, K] in the kernel's k order.  The fp16 x fp16 products are exact in fp32; the accumulator takes them
    ACC_CHUNK at a time and each update is off by at most 2^-23 (one fp32 ulp: truncation allowed as well as
    round-to-nearest) of |previous partial sum| + sum |products of the chunk|.  The partial sums are computed in fp64."""
    s = torch.zeros(*a.shape[:-1], w.shape[-2], dtype=F64, device=a.device)
    tot = torch.zeros_like(s)
    for k0 in range(0, a.shape[-1], ACC_CHUNK):
        ab, wb = a[..., k0:k0 + ACC_CHUNK], w[..., k0:k0 + ACC_CHUNK].transpose(-1, -2)
        tot += s.abs() + ab.abs() @ wb.abs()
        s += ab @ wb
    return tot * 2.0 ** -23


def split_product_bound(x, w):
    """|x w^T - (x_hi w_hi + x_lo w_hi + x_hi w_lo)^T| summed over k, for fp32 x [M, K] and w [N, K] split by split16.
    With x = x_hi + x_lo + e_x and w = w_hi + w_lo + e_w (all exact in fp64):
    x w - P3 = x_lo w_lo + e_x w + x e_w - e_x e_w."""
    xh, xl = (t.double() for t in split16(x))
    wh, wl = (t.double() for t in split16(w))
    x64, w64 = x.double(), w.double()
    ex, ew = x64 - xh - xl, w64 - wh - wl
    return (xl.abs() @ wl.abs().t() + ex.abs() @ w64.abs().t() + x64.abs() @ ew.abs().t() + ex.abs() @ ew.abs().t())


def check(name, err, bound, mutants, where=None):
    """Assert err <= bound everywhere and that every mutant's error exceeds the bound by MUTANT_MARGIN somewhere; print
    the ratios.  err, bound, mutant errors: fp64 tensors of one shape; where: elements to compare (default all)."""
    if where is not None:
        err, bound = err[where], bound[where]
        mutants = {k: v[where] for k, v in mutants.items()}
    ratio = err / bound
    r = ratio.max().item() if ratio.numel() else 0.0
    msg = ["%s: kernel error / bound = %.3g" % (name, r)]
    bad = []
    for mname, merr in mutants.items():
        mr = (merr / bound).max().item()
        msg.append("  mutant %-38s error / bound = %.3g" % (mname + ":", mr))
        if not mr >= MUTANT_MARGIN:
            bad.append(mname)
    print("\n".join(msg))
    assert torch.isfinite(err).all(), "%s: non-finite output" % name
    assert r <= 1.0, "%s: kernel error %.3g x the bound (worst element %d)" % (name, r, int(ratio.argmax()))
    assert not bad, "%s: the bound does not discriminate %s" % (name, bad)


def grid_operands(M, N, K, g):
    """fp16 A [M, K] = i/8 (|i| <= 16, narrowed to 16384 / K above K = 1024), W [N, K] = j/256 (|j| <= 8): every product
    is a multiple of 2^-11 and every partial sum a multiple of 2^-11 below 2^6 -- 17 bits, exact in fp32 in any order.
    The accumulation is then exact and the bounds below are the epilogue's alone."""
    assert K <= 2048
    imax = min(16, 16384 // K)
    a = (torch.randint(-imax, imax + 1, (M, K), device="cuda", generator=g).float() / 8).half()
    w = (torch.randint(-8, 9, (N, K), device="cuda", generator=g).float() / 256).half()
    return a, w


def gelu64(x):
    return 0.5 * x * torch.special.erfc(-x / math.sqrt(2.0))


def gelu_tanh64(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def gelu_bound(g):
    """|hi + lo - gelu(x)| for the fp32 x the epilogue sees: gelu_erf's 8e-7 plus 2^-22 |gelu| (its fp32 rounding
    and the hi + lo split)."""
    return GELU_ABS + 2.0 ** -22 * g.abs()


def run_gemm_epi(a, w, bias, N, epi):
    L, lib = _lib()
    M, K = a.shape
    out = torch.full((M, 2 * N if epi == 0 else N), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_gemm_epi(_p(a), _p(w), _p(bias), _p(out), M, N, K, epi, _stream()))
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------ EpiBiasF16Wide<GELU>
@pytest.mark.parametrize("M", [15360, 300])
def test_wide_gelu_ffn_up(M):
    """The DiP FFN up-projection epilogue (M = 2 x 128 x 60 tokens, N = ff = 1024, K = 2d = 1024): hi + lo against fp64
    gelu(A W^T + b).  The fp32 bias add costs |gelu'| <= 1.13 times 2^-24 |x|."""
    N, K = 1024, 1024
    g = torch.Generator(device="cuda").manual_seed(M)
    a, w = grid_operands(M, N, K, g)
    bias = torch.randn(N, device="cuda", generator=g)
    out = run_gemm_epi(a, w, bias, N, 0)
    x = a.double() @ w.double().t() + bias.double()
    ref = gelu64(x)
    hi, lo = out[:, :N].double(), out[:, N:].double()
    bound = gelu_bound(ref) + 2.0 ** -23 * x.abs()
    check("EpiBiasF16Wide<GELU> M=%d" % M, (hi + lo - ref).abs(), bound,
          {"lo half zeroed": (hi - ref).abs(), "tanh-GELU": (gelu_tanh64(x) - ref).abs()})


def test_gelu_sweep():
    """gelu_erf over all x through the Wide epilogue: W = I (N = K = 1024), A an fp16 grid of [-6, 6] at 2^-8, fp32
    bias offsets, so the epilogue sees x = fp32(a + b) exactly: [-6, 6] densely (60 columns per grid step) and, from
    64 columns biased by -5.5 - U(0, 1000), everything down to about -1008."""
    M, N = 3072, 1024
    g = torch.Generator(device="cuda").manual_seed(5)
    grid = torch.arange(-6 * 256, 6 * 256 + 1, device="cuda", dtype=torch.float32) / 256
    idx = (torch.arange(M * N, device="cuda", dtype=torch.int64) * 7919) % grid.numel()
    a = grid[idx].view(M, N).half()
    w = torch.eye(N, device="cuda").half()
    bias = torch.rand(N, device="cuda", generator=g) / 256
    bias[-64:] = -5.5 - 1000 * torch.rand(64, device="cuda", generator=g)
    out = run_gemm_epi(a, w, bias, N, 0)
    x = (a.float() + bias).double()                       # the accumulator is a exactly; the bias add is the epilogue's
    ref = gelu64(x)
    err = (out[:, :N].double() + out[:, N:].double() - ref).abs()
    bound = gelu_bound(ref)
    over = err > bound
    if over.any():
        xs = x[over]
        print("gelu sweep: %d elements over the bound, x in [%.4g, %.4g]; worst at x = %.6g (error %.3g)" % (
            int(over.sum()), xs.min().item(), xs.max().item(), x.flatten()[int((err / bound).argmax())].item(),
            err.max().item()))
    print("gelu sweep: x in [%.4g, %.4g], %d values below -5.5" % (x.min().item(), x.max().item(), int((x < -5.5).sum())))
    check("gelu_erf sweep", err, bound, {"tanh-GELU": (gelu_tanh64(x) - ref).abs()})


# ------------------------------------------------------------------------------------------------ EpiBiasF16Global
@pytest.mark.parametrize("M", [4096, 120])
def test_global_bias_kv_projection(M):
    """The DiP K/V projection of all layers at once (N = 8 layers x 2d = 8192 > the 2048-column staged-bias limit, K = d):
    fp16(A W^T + b) within half an fp16 ulp plus the fp32 bias add.  The bias differs per column, so a chunk that reads
    another chunk's bias is caught."""
    N, K = 8192, 512
    g = torch.Generator(device="cuda").manual_seed(M + 1)
    a, w = grid_operands(M, N, K, g)
    bias = torch.randn(N, device="cuda", generator=g)
    out = run_gemm_epi(a, w, bias, N, 1)
    y = a.double() @ w.double().t()
    ref = y + bias.double()
    bound = half_ulp16(ref) + U32 * ref.abs()
    shifted = y + bias.double().roll(-32)
    check("EpiBiasF16Global M=%d" % M, (out.double() - ref).abs(), bound,
          {"bias shifted by one 32-column chunk": (shifted.float().half().double() - ref).abs()})


# ------------------------------------------------------------------------------------------------ EpiEmbed
@pytest.mark.parametrize("B,JF,T,s_off,halves", [
    (3, 263, 24, 1, 2),       # encoder, CFG: B*S = 75 rows, one partial tile
    (64, 263, 196, 1, 2),     # HumanML3D at batch 64: B*S = 12608 = 98.5 tiles
    (4, 150, 60, 1, 1),       # a2m (HumanAct12 features), no CFG
    (2, 263, 40, 20, 2),      # DiP: 20 prefix rows per sequence
])
def test_embed(B, JF, T, s_off, halves):
    """pack_input -> split_weight -> pe_bias -> EpiEmbed GEMM: hi + lo of the residual stream against fp64
    x W^T + b + pe[s] (rows s < s_off: b + pe[s]); the two CFG copies bit-identical."""
    L, lib = _lib()
    d = 512
    S = T + s_off
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + JF + s_off)
    x = torch.randn(B, JF, T, device="cuda", generator=g)
    w = torch.randn(d, JF, device="cuda", generator=g) / JF ** 0.5
    b = torch.randn(d, device="cuda", generator=g) * 0.1
    pe = torch.randn(S + 3, d, device="cuda", generator=g) * 0.5
    hres = torch.full((halves * B * S, 2 * d), float("nan"), device="cuda", dtype=torch.float16)
    L.check(lib.b200mdm_test_embed(_p(x), _p(w), _p(b), _p(pe), _p(hres), B, JF, T, d, s_off, halves, _stream()))
    torch.cuda.synchronize()
    MB = B * S
    if halves == 2:
        assert torch.equal(hres[:MB].view(torch.int16), hres[MB:].view(torch.int16)), "CFG copies differ"
    got = hres[:MB, :d].double() + hres[:MB, d:].double()
    ref, bound, mutants = embed_reference(x, w, b, pe, s_off)
    check("embed B=%d JF=%d T=%d s_off=%d halves=%d" % (B, JF, T, s_off, halves), (got - ref).abs(), bound, mutants)


def embed_reference(x, w, b, pe, s_off):
    """(fp64 x W^T + b + pe[s] of the GEMM rows (b, s), its per-element bound, errors of the mutants) for the embedding
    hook's inputs x [B, JF, T], w [d, JF], b [d], pe; the operands as the kernel splits them, [hi | lo | hi] x
    [hi | hi | lo] with zero pad columns up to Kp = ceil8(JF)."""
    B, JF, T = x.shape
    S, Kp = T + s_off, (JF + 7) // 8 * 8
    MB = B * S
    xr = torch.zeros(B, S, JF, device="cuda")                   # GEMM rows (b, s); frame t at s = s_off + t
    xr[:, s_off:] = x.transpose(1, 2)
    xr = xr.view(MB, JF)
    s_idx = torch.arange(MB, device="cuda") % S
    bpe = b.double() + pe.double()[:S]                           # [S, d]
    ref = xr.double() @ w.double().t() + bpe[s_idx]

    def padk(t):
        return torch.nn.functional.pad(t.double(), (0, Kp - JF))
    xh, xl = split16(xr)
    wh, wl = split16(w)
    a3 = torch.cat([padk(xh), padk(xl), padk(xh)], 1)            # the kernel's operands, [hi | lo | hi] x [hi | hi | lo]
    w3 = torch.cat([padk(wh), padk(wh), padk(wl)], 1)
    p3 = a3 @ w3.t() + bpe[s_idx]
    # split truncation + accumulation + fp32 pe_bias and epilogue adds + the [hi | lo] store (2^-22 relative, 2^-25 floor)
    bound = (split_product_bound(xr, w) + acc_bound(a3, w3) + U32 * bpe.abs()[s_idx] + (U32 + 2.0 ** -22) * ref.abs()
             + 2.0 ** -25)
    pe_prev = b.double() + pe.double()[(s_idx - 1).clamp(min=0)]
    return ref, bound, {"A_lo W_hi dropped": (p3 - padk(xl) @ padk(wh).t() - ref).abs(),
                        "A_hi W_lo dropped": (p3 - padk(xh) @ padk(wl).t() - ref).abs(),
                        "pe row s-1": (p3 - bpe[s_idx] + pe_prev - ref).abs()}


# ------------------------------------------------------------------------------------------------ EpiOutStep
SCHED_ROW = [0.31, 0.68, 0.11, 1.07, 0.37, 0.93, 0.42, 0.06]   # c1 c2 sig_ddpm sr srm1 sqrt_abp coef_eps sig_ddim
CONST_NOISE, CLIP = 1, 2


def _step_f32(mode, x0, xt, nz, row, fma=False):
    """x_out in the kernel's op order, numpy float32 (every op rounded); fma=True: the contracted variant."""
    f = np.float32
    c1, c2, sgp, sr, srm1, sq, ce, sgi = (f(v) for v in row)
    if mode == 0:
        return x0.copy()
    if not fma:
        if mode == 1:
            return (c1 * x0 + c2 * xt) + sgp * nz
        eh = (sr * xt - x0) / srm1
        return (x0 * sq + ce * eh) + sgi * nz
    d = np.float64

    def fmaf(a, b, c):
        return (d(a) * d(b) + d(c)).astype(np.float32)
    if mode == 1:
        return fmaf(sgp, nz, fmaf(c1, x0, c2 * xt))
    eh = fmaf(sr, xt, -x0) / srm1
    return fmaf(sgi, nz, fmaf(x0, sq, ce * eh))


@pytest.mark.parametrize("mode,halves,JF,B,T,s_off,flags,inpaint,alias", [
    (0, 1, 263, 3, 24, 1, 0, False, False),
    (1, 2, 263, 4, 24, 1, 0, False, True),              # scales 0, 1, 2.5, 7.5; x_out aliases x_t (the loop)
    (2, 2, 263, 4, 45, 1, CONST_NOISE, False, True),
    (1, 2, 150, 4, 60, 1, CLIP, False, False),          # a2m features, clip_denoised
    (2, 1, 150, 3, 60, 1, 0, True, False),              # inpainting
    (1, 2, 263, 4, 40, 20, CLIP | CONST_NOISE, True, True),   # DiP prefix rows
    (2, 2, 263, 64, 196, 1, 0, False, True),            # HumanML3D batch 64: B*T = 12544 frame rows
])
def test_out_step(mode, halves, JF, B, T, s_off, flags, inpaint, alias):
    """blend_split -> split-weight EpiOutStep GEMM: pred_xstart against fp64 blend -> projection of the residual stream;
    x_out bit for bit against a float32 evaluation of the sampler update from the returned pred_xstart."""
    L, lib = _lib()
    d = 512
    S = T + s_off
    g = torch.Generator(device="cuda").manual_seed(mode * 7 + halves * 3 + JF + B + T)
    h = torch.randn(halves * B * S, d, device="cuda", generator=g) * 1.2
    hh, hl = split16(h)
    hres = torch.cat([hh, hl], 1).contiguous()
    scale = torch.tensor([[0.0, 1.0, 2.5, 7.5][i % 4] for i in range(B)], device="cuda") if halves == 2 else None
    w = torch.randn(JF, d, device="cuda", generator=g) / d ** 0.5
    b = torch.randn(JF, device="cuda", generator=g) * 0.1
    xt0 = torch.randn(B, JF, T, device="cuda", generator=g)
    noise = torch.randn(1 if flags & CONST_NOISE else B, JF, T, device="cuda", generator=g)
    row = torch.tensor(SCHED_ROW, device="cuda")
    mask = (torch.rand(B, JF, T, device="cuda", generator=g) < 0.3) if inpaint else None
    motion = (torch.rand(B, JF, T, device="cuda", generator=g) * 1.8 - 0.9) if inpaint else None
    xt = xt0.clone()
    xout = xt if alias else torch.full_like(xt0, float("nan"))
    pred = torch.full_like(xt0, float("nan"))
    L.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w), _p(b), _p(xt), _p(noise), _p(row), mode, flags,
                                      _p(mask.to(torch.uint8) if inpaint else None), _p(motion), _p(xout), _p(pred),
                                      B, JF, T, d, s_off, halves, _stream()))
    torch.cuda.synchronize()

    ref, bound, v_swapped, vl, wh = out_reference(hh, hl, scale, w, b, B, T, s_off, halves)

    def to_bjt(t):
        return t.view(B, T, JF).permute(0, 2, 1)

    def post(t):                                                   # inpainting, then clip_denoised (the kernel's order)
        t = to_bjt(t)
        if inpaint:
            t = torch.where(mask, motion.double(), t)
        return t.clamp(-1, 1) if flags & CLIP else t
    ref_p = post(ref)
    mutants = {"A_lo W_hi dropped": (post(ref - vl @ wh.t()) - ref_p).abs()}
    if halves == 2:
        mutants["scale applied to the uncond half"] = (post(v_swapped @ w.double().t() + b.double()) - ref_p).abs()
    keep = ~mask if inpaint else None
    check("out step mode=%d halves=%d JF=%d B=%d T=%d flags=%d" % (mode, halves, JF, B, T, flags),
          (pred.double() - ref_p).abs(), to_bjt(bound), mutants, where=keep)
    if inpaint:
        assert torch.equal(pred[mask], motion[mask]), "inpainted elements must equal the motion exactly"
    if flags & CLIP:
        assert pred.abs().max().item() <= 1.0
    check_x_out(mode, pred, xt0, noise, xout)


def check_x_out(mode, pred, xt0, noise, xout, row=SCHED_ROW):
    """x_out bit for bit against the float32 update evaluated from the pred_xstart the kernel returned, with schedule
    row `row`; an FMA-contracted evaluation must differ somewhere."""
    x0n, xtn = pred.cpu().numpy(), xt0.cpu().numpy()
    nzn = np.broadcast_to(noise.cpu().numpy(), xtn.shape)
    want = _step_f32(mode, x0n, xtn, nzn, row)
    gotx = xout.cpu().numpy()
    diff = int((gotx.view(np.int32) != want.view(np.int32)).sum())
    line = "  x_out: %d of %d elements differ from the float32 evaluation" % (diff, want.size)
    if mode != 0:
        fm = _step_f32(mode, x0n, xtn, nzn, row, fma=True)
        nfm = int((fm.view(np.int32) != want.view(np.int32)).sum())
        line += "; FMA-contracted mutant differs in %d" % nfm
        assert nfm > 0, "the bit-exact check would not see an FMA-contracted update"
    print(line)
    assert diff == 0


def out_reference(hh, hl, scale, w, b, B, T, s_off, halves):
    """(fp64 model output [B*T, JF] of the frame rows of the residual stream hh + hl (both CFG halves), its per-element
    bound, the blend with the scale on the unconditional half, the lo part of the blend's split and the hi part of W's)
    for the output hooks."""
    S = T + s_off
    # frame rows of the residual stream: (b, t) -> row b*S + s_off + t of each CFG half
    rows = (torch.arange(B, device="cuda")[:, None] * S + s_off + torch.arange(T, device="cuda")[None, :]).flatten()
    c = (hh.double() + hl.double())[rows]
    s = torch.zeros(B * T, 1, dtype=F64, device="cuda")
    if halves == 2:
        u = (hh.double() + hl.double())[B * S + rows]
        s = scale.double().repeat_interleave(T)[:, None]
        v = u + s * (c - u)
        v_swapped = c + s * (u - c)                                # scale applied to the uncond half
    else:
        u, v, v_swapped = c, c, None
    w64 = w.double()
    ref = v @ w64.t() + b.double()                                 # [B*T, JF]
    # the fp32 blend (three roundings: |dv| <= 2^-24 (2 |s| |c - u| + |v|)), the fp16 [hi|lo|hi] x [hi|hi|lo] split of
    # v (|lo| <= 2^-11 |v|, |v - hi - lo| <= 2^-22 |v| + 2^-25) and of W, the accumulation, the fp32 bias add
    V = v.abs() * (1 + 2.0 ** -20)
    wh, wl = (t.double() for t in split16(w))
    ew = w64 - wh - wl
    dv = U32 * (2 * s.abs() * (c - u).abs() + V) * 1.01
    vh, vl = (t.double() for t in split16(v.float()))
    a3 = torch.cat([vh, vl, vh], 1)
    w3 = torch.cat([wh, wh, wl], 1)
    bound = ((dv + 2.0 ** -22 * V + 2.0 ** -25) @ w64.abs().t() + (2.0 ** -11 * 1.001 * V) @ wl.abs().t()
             + V @ ew.abs().t() + acc_bound(a3, w3) + U32 * (ref.abs() + 1e-30))
    return ref, bound, v_swapped, vl, wh
