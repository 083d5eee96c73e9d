"""GPU: the fused residual + LayerNorm GEMM moves the residual stream only with TMA loads and stores, so its row tails
rely on the tensor map's extent (loads zero-filled, stores clipped at row M).  Here the [hi | lo] stream is a view into a
larger buffer with guard rows before and after it: the result must match torch fp32 and no guard row may change."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 96   # rows on each side: more than one 64-row store box


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("M,K", [
    (77, 1024),        # one tile, second warpgroup's rows wholly past M
    (130, 512),        # two live rows in the last tile
    (200, 512),        # last tile: first warpgroup partly live, second wholly past M
    (300, 1024),       # last tile: second warpgroup partly live
    (25216 // 4, 512), # several tiles per cluster, last one partial (6304 = 49 * 128 + 32)
])
def test_gemm_resid_ln_guard_rows(M, K):
    from b200mdm import _lib as L
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(3 * M + K)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    w = (torch.randn(512, K, device="cuda", generator=g) / K ** 0.5).half()
    bias = torch.randn(512, device="cuda", generator=g) * 0.1
    gamma = 1 + 0.1 * torch.randn(512, device="cuda", generator=g)
    beta = 0.1 * torch.randn(512, device="cuda", generator=g)
    h = torch.randn(M, 512, device="cuda", generator=g) * 1.5 + 0.2
    hi = h.half()
    buf = torch.randn(GUARD + M + GUARD, 1024, device="cuda", generator=g).half()
    hres = buf[GUARD:GUARD + M]
    hres[:, :512] = hi
    hres[:, 512:] = (h - hi.float()).half()
    before = buf.clone()
    h_in = hres[:, :512].float() + hres[:, 512:].float()
    ref = torch.nn.functional.layer_norm(h_in + a.float() @ w.float().t() + bias, (512,), gamma, beta, 1e-5)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.b200mdm_test_gemm_resid_ln(_p(a), _p(w), _p(bias), _p(gamma), _p(beta), _p(hres), M, K, stream))
    torch.cuda.synchronize()
    assert torch.equal(buf[:GUARD].view(torch.int16), before[:GUARD].view(torch.int16)), "rows before the stream changed"
    assert torch.equal(buf[GUARD + M:].view(torch.int16), before[GUARD + M:].view(torch.int16)), "rows after row M changed"
    out = hres[:, :512].float() + hres[:, 512:].float()
    assert torch.isfinite(out).all()
    assert (out - ref).abs().max().item() < 2e-4
