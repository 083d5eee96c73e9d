"""CPU: the wiring mutants of the guided DDPM / DDIM step (tests/test_guided_step_gpu.py) can be seen on their cases.

For every case of tests/guided_step_cases.py and every step it runs, the fp32 oracle denoiser's x0 stands in for the
engine's; the correct guided x0 (fp64 oracle, then inpainting and the clamp) and each mutant's are formed in fp64, and
every mutant must differ from the correct one by at least 8 times the bound the GPU file holds the kernel to,
2^-12 max |guided - x0| + 2 u K max |x0|.  A mutant that the GPU file then fails to separate from the engine's bits
means a weak case, and this file catches it first."""
import pytest
import torch

import b200mdm
import guided_step_cases as gc


def mutant_x0(k, g, x0, order):
    """the pred_xstart of guidance inputs g on x0 [n, D, 1, T] in tail order `order`, fp64"""
    rows = k.idx
    if order == "after_inpaint":
        out, _ = gc.guide64(k, gc.inpaint(k, x0.double(), rows, True), g)
        return gc.clamp(k, out)
    if order == "after_clamp":
        out, _ = gc.guide64(k, gc.clamp(k, gc.inpaint(k, x0.double(), rows, True)), g)
        return out
    out, _ = gc.guide64(k, x0, g)
    return gc.clamp(k, gc.inpaint(k, out, rows, True))


@pytest.mark.parametrize("name", list(gc.CASES) + list(gc.HEADLINE))
def test_mutants_miss_the_bound(name):
    c = dict(gc.CASES, **gc.HEADLINE)[name]
    k = gc.build(c)
    _, sdkw = gc.model_args(c)
    sd = b200mdm.synthetic_state_dict(**sdkw)
    rows = k.idx
    den = gc.oracle_denoiser(k, sd, rows)
    cond = gc.oracle_denoiser(k, sd, rows, scale=torch.ones(k.B))
    base = gc.guide_inputs(k)
    muts = gc.mutants(k)
    assert muts, name
    for sampler, eta, i in c["steps_run"]:
        with torch.no_grad():
            x0 = den(k.xt[rows], i)
            x0c = cond(k.xt[rows], i) if "cond_x0" in muts else None
        want, _ = gc.guide64(k, x0, base)
        bnd = gc.bound(k, x0, want, k.iters)
        pred = gc.clamp(k, gc.inpaint(k, want, rows, True))
        print("%s %s eta %.1f i %d: lambda %.3g, |dx| %.3g, bound %.3g"
              % (name, sampler, eta, i, k.step, float((want - x0.reshape(want.shape).double()).abs().max()), bnd))
        for m, (g, src, order) in muts.items():
            got = mutant_x0(k, g, x0c if src == "cond" else x0, order)
            miss = float((got.reshape(pred.shape) - pred).abs().max()) / bnd
            print("   mutant %-20s misses the bound %.1f-fold" % (m, miss))
            assert miss >= gc.MISS, (name, i, m, miss)
