"""GPU: the ping-pong projection GEMM (gemm_pingpong.cuh) at the tile schedules the other tests do not reach, against
fp64 with the criteria of test_gemm_tcgen05 / test_wide_gelu_ffn_up / test_global_bias_kv_projection.

The two consumer warpgroups take the CTA's tiles in turn (i even / odd), so the schedules of interest are: an odd
number of tiles per CTA (one warpgroup runs one more tile than the other), one tile per CTA (the second warpgroup
has none), and long launches in which the operand ring wraps many times and the two warpgroups hand it back and forth
at every tile.  Tile counts below assume the 132 SMs of an H100 SXM; on another part the shapes still run, only the
per-CTA counts differ."""
import pytest
import torch

from test_epilogues_gpu import (U32, check, gelu64, gelu_bound, gelu_tanh64, grid_operands, half_ulp16, run_gemm_epi)
from test_kernels_gpu import run_gemm_f16

pytestmark = pytest.mark.gpu


def _bias(N, g):
    # one bias per 12 / N stratum of [-6, 6]: every launch crosses the whole GELU
    return -6 + 12 * (torch.randperm(N, device="cuda", generator=g).float() + torch.rand(N, device="cuda", generator=g)) / N


@pytest.mark.parametrize("M,N,K,act", [
    (25216, 1536, 512, 0),   # c2 QKV: 197 x 12 = 2364 tiles, 17 or 18 per CTA
    (25216, 1024, 512, 1),   # c2 FFN-up + GELU: 1576 tiles, 11 or 12 per CTA
    (1408, 1536, 512, 0),    # 132 tiles: exactly one per CTA, the second warpgroup idle
    (1408, 1536, 512, 1),
    (2816, 1536, 512, 0),    # 264 tiles: one per warpgroup
    (1500, 1000, 320, 1),    # 12 x 8 = 96 tiles (fewer CTAs than SMs), M and N tails, 5 k-blocks (ring wraps mid-tile)
    (3000, 1536, 64, 0),     # one k-block per tile: four tiles share one lap of the ring
    (640, 136, 1024, 0),     # 5 x 2 tiles; the second column tile holds 8 live columns
])
def test_pingpong_f16(M, N, K, act):
    """EpiBiasF16<act> through b200mdm_test_gemm_f16(block_n = 128).  act = 0: fp16(fp32(acc + bias)) bit for bit;
    act = 1: against fp64 gelu(acc + bias) within half an fp16 ulp + gelu_erf's bound + the fp32 bias add."""
    g = torch.Generator(device="cuda").manual_seed(M * 5 + N * 11 + K + act)
    a, w = grid_operands(M, N, K, g)
    bias = _bias(N, g)
    out = run_gemm_f16(a, w, bias, act, 128)
    acc = a.double() @ w.double().t()
    if not act:
        want = (acc.float() + bias).half()
        diff = int((out.view(torch.int16) != want.view(torch.int16)).sum())
        nb16 = int(((acc.float() + bias.half().float()).half().view(torch.int16) != want.view(torch.int16)).sum())
        print("ping-pong f16 M=%d N=%d K=%d: %d of %d elements differ from fp16(fp32(acc + bias)); the fp16-bias "
              "mutant differs in %d" % (M, N, K, diff, want.numel(), nb16))
        assert nb16 > 0, "the bit-exact check would not see an fp16 bias"
        assert diff == 0
        return
    x = acc + bias.double()
    ref = gelu64(x)
    bound = half_ulp16(ref) + gelu_bound(ref) + 1.13 * U32 * x.abs()
    check("ping-pong EpiBiasF16<GELU> M=%d N=%d K=%d" % (M, N, K), (out.double() - ref).abs(), bound, {
        "tanh-GELU": (gelu_tanh64(x) - ref).abs(),
        "bias rounded to fp16": (gelu64(acc + bias.half().double()) - ref).abs(),
        "bias of the next 32-column chunk": (gelu64(acc + bias.double().roll(-32)) - ref).abs(),
    })


@pytest.mark.parametrize("M", [
    17024,   # 133 x 8 = 1064 tiles: 8 CTAs run 9 (odd), the rest 8
    1024,    # 64 tiles, one per CTA
])
def test_pingpong_wide_gelu(M):
    """EpiBiasF16Wide<GELU> (the DiP FFN-up, K = 2d = 1024: 16 k-blocks per tile) -- hi + lo against fp64 gelu."""
    N, K = 1024, 1024
    g = torch.Generator(device="cuda").manual_seed(M + 3)
    a, w = grid_operands(M, N, K, g)
    bias = torch.randn(N, device="cuda", generator=g)
    out = run_gemm_epi(a, w, bias, N, 0)
    x = a.double() @ w.double().t() + bias.double()
    ref = gelu64(x)
    hi, lo = out[:, :N].double(), out[:, N:].double()
    bound = gelu_bound(ref) + 2.0 ** -23 * x.abs()
    check("ping-pong EpiBiasF16Wide<GELU> M=%d" % M, (hi + lo - ref).abs(), bound,
          {"lo half zeroed": (hi - ref).abs(), "tanh-GELU": (gelu_tanh64(x) - ref).abs(),
           "bias of the next 64-column slab": (gelu64(x - bias.double() + bias.double().roll(-64)) - ref).abs()})


@pytest.mark.parametrize("M,N", [
    (4096, 8192),   # the DiP all-layer K/V projection: 32 x 64 = 2048 tiles, 15 or 16 per CTA
    (5000, 8160),   # 40 x 64 = 2560 tiles, 19 or 20 per CTA; the last column tile ends inside a 64-column slab
])
def test_pingpong_global_bias(M, N):
    """EpiBiasF16Global (bias read per tile from global memory, N > 2048): fp16(A W^T + b) within half an fp16 ulp
    plus the fp32 bias add."""
    K = 512
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a, w = grid_operands(M, N, K, g)
    bias = torch.randn(N, device="cuda", generator=g)
    out = run_gemm_epi(a, w, bias, N, 1)
    y = a.double() @ w.double().t()
    ref = y + bias.double()
    bound = half_ulp16(ref) + U32 * ref.abs()
    check("ping-pong EpiBiasF16Global M=%d N=%d" % (M, N), (out.double() - ref).abs(), bound,
          {"bias shifted by one 32-column chunk": ((y + bias.double().roll(-32)).float().half().double() - ref).abs(),
           "bias of the other warpgroup's tile": ((y + bias.double().roll(-128)).float().half().double() - ref).abs()})
