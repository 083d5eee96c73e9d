"""CPU: multistep DPM-Solver++ (data prediction; Lu et al. 2022, Algorithm 2) -- the engine's coefficient table against
the fp64 formulas, the order-1 oracle against DDIM at eta = 0, the solver's convergence order on a Gaussian data
distribution whose probability-flow ODE has a closed-form solution, and the argument checks of the Python API and of
the C ABI that run before any device work."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args
from oracle import dpm_oracle as do
from oracle import mdm_oracle as mo
from oracle import schedule_oracle as so


def _diffusion(name, steps, respacing=None):
    betas = gd.get_named_beta_schedule(name, steps)
    kw = dict(betas=betas, model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL,
              loss_type=gd.LossType.MSE)
    if respacing is None:
        return gd.GaussianDiffusion(**kw)
    return rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(steps, respacing), **kw)


SCHEDULES = [("linear", 1000, None), ("cosine", 1000, None), ("cosine", 1000, "ddim10"), ("cosine", 1000, [10, 15, 20]),
             ("cosine", 50, None)]


@pytest.mark.parametrize("name,steps,respacing", SCHEDULES)
def test_table_against_fp64_formulas(name, steps, respacing):
    d = _diffusion(name, steps, respacing)
    rows = d.schedule_dpm_rows()
    n = d.num_timesteps
    assert rows.dtype == np.float32 and rows.shape == (n, _lib.SCHED_DPM_STRIDE)
    tables = {"alphas_cumprod": d.alphas_cumprod, "alphas_cumprod_prev": d.alphas_cumprod_prev}
    ref = do.dpm_table(tables)
    # one rounding of the fp64 value (the two fp64 restatements differ far below an fp32 ulp)
    assert np.all(np.abs(rows.astype(np.float64) - ref) <= np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)), \
        np.abs(rows - ref).max()
    assert rows[0].tolist() == [0.0, 1.0, 1.0, 0.0]
    lam = do.log_snr(d.alphas_cumprod)
    assert np.all(np.diff(lam) < 0)                           # lambda strictly increasing toward i = 0
    # c_cur + c_prev = c0 (D is an affine combination of the two x0), and the first-order row is DDIM at eta = 0
    np.testing.assert_allclose(ref[:, 2] + ref[:, 3], ref[:, 1], rtol=1e-12, atol=1e-15)
    ab, abp = d.alphas_cumprod, d.alphas_cumprod_prev
    np.testing.assert_allclose(ref[1:, 1], np.sqrt(abp[1:]) - np.sqrt(ab[1:]) * np.sqrt(1 - abp[1:]) / np.sqrt(1 - ab[1:]),
                               rtol=1e-9)


def test_order1_oracle_is_ddim_eta0():
    """Every step of the fp64 order-1 oracle equals reference DDIM at eta = 0 (mdm_oracle.ddim_step) to fp64 rounding."""
    tabs = so.diffusion_tables(so.respaced(so.named_betas("cosine", 1000), so.space_timesteps(1000, "ddim10"))[0])
    g = torch.Generator().manual_seed(3)
    W = torch.randn(64, 64, generator=g, dtype=torch.float64) / 8
    denoise = lambda x, i: torch.tanh(x @ W) * 0.9 + 0.05 * i
    x_T = torch.randn(4, 64, generator=g, dtype=torch.float64)
    got = []
    do.dpm_loop(denoise, tabs, x_T, order=1, f64=True, collect=got)
    x = x_T.clone()
    n = len(tabs["betas"])
    assert len(got) == n
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = denoise(x, i)
        e = (np.sqrt(1.0 / tabs["alphas_cumprod"][i]) * x - x0) / np.sqrt(1.0 / tabs["alphas_cumprod"][i] - 1)
        x = x0 * np.sqrt(tabs["alphas_cumprod_prev"][i]) + np.sqrt(1 - tabs["alphas_cumprod_prev"][i]) * e
        assert torch.allclose(got[k][0], x, rtol=1e-12, atol=1e-12), (k, (got[k][0] - x).abs().max())
        assert torch.allclose(got[k][1], x0, rtol=0, atol=0)
        x = got[k][0]
    # and the fp32 reference step of the oracles agrees to fp32 rounding
    x = x_T.float()
    x0 = denoise(x.double(), n - 1).float()
    ref = mo.ddim_step(tabs, x0, x, n - 1, torch.zeros_like(x))
    row = do.dpm_table(tabs)[n - 1].astype(np.float32)
    np.testing.assert_allclose(do.update32(row, x.numpy(), x0.numpy()), ref.numpy(), rtol=1e-5, atol=1e-6)


# Convergence on N(mu, s^2 I): exact denoiser x0(x, i) = mu + alpha s^2 / (alpha^2 s^2 + sigma^2) (x - alpha mu); the
# probability-flow ODE maps x_T to mu + s (x_T - alpha_T mu) / sqrt(alpha_T^2 s^2 + sigma_T^2).  Unit-variance data, like
# MDM's normalised features.  Measured endpoint errors (Frobenius-relative, fp64, DESIGN.md section 2):
#   N        10        20        40        80
#   order 1  1.23e-1   6.00e-2   2.97e-2   1.48e-2    ratios 2.04 2.02 2.01
#   order 2  1.08e-1   2.51e-2   5.24e-3   1.07e-3    ratios 4.29 4.79 4.91
MU, S = 0.3, 1.0


def _gaussian_errors(order):
    x_T = torch.from_numpy(np.random.default_rng(1).standard_normal(4096))
    errs = []
    for N in (10, 20, 40, 80):
        betas, _, _ = so.respaced(so.named_betas("cosine", 1000), so.space_timesteps(1000, str(N)))
        tabs = so.diffusion_tables(betas)
        ac = tabs["alphas_cumprod"]

        def denoise(x, i):
            a, v = np.sqrt(ac[i]), 1.0 - ac[i]
            return MU + a * S * S / (a * a * S * S + v) * (x - a * MU)
        aT, vT = np.sqrt(ac[-1]), 1.0 - ac[-1]
        exact = MU + S * (x_T - aT * MU) / np.sqrt(aT * aT * S * S + vT)
        out = do.dpm_loop(denoise, tabs, x_T, order=order, f64=True)
        errs.append(float((out - exact).norm() / exact.norm()))
    return errs


def test_convergence_order_on_gaussian_data():
    e1, e2 = _gaussian_errors(1), _gaussian_errors(2)
    r1 = [a / b for a, b in zip(e1, e1[1:])]
    r2 = [a / b for a, b in zip(e2, e2[1:])]
    print("order 1 errors %s ratios %s" % (" ".join("%.3e" % e for e in e1), " ".join("%.2f" % r for r in r1)))
    print("order 2 errors %s ratios %s" % (" ".join("%.3e" % e for e in e2), " ".join("%.2f" % r for r in r2)))
    assert all(1.8 < r < 2.3 for r in r1), r1
    assert all(r > 3.5 for r in r2[1:]) and r2[0] > 3.0, r2
    assert all(b < a for a, b in zip(e1, e2)), (e1, e2)


# ---------------------------------------------------------------------------------------------------------------------
def test_arguments_checked_before_any_device_work(monkeypatch):
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=6),
                                                          SimpleNamespace(dataset=SimpleNamespace()))

    def no_engine(*a, **k):
        raise AssertionError("the engine was reached")
    monkeypatch.setattr(type(diffusion), "_prepare", no_engine)
    shape = (2, 263, 1, 24)
    loop = diffusion.dpm_solver_sample_loop
    prog = lambda *a, **k: next(diffusion.dpm_solver_sample_loop_progressive(*a, **k))
    for fn in (loop, prog):
        with pytest.raises(NotImplementedError):
            fn(model, shape, denoised_fn=lambda v: v)
        with pytest.raises(NotImplementedError):
            fn(model, shape, cond_fn=lambda *a: 0)
        with pytest.raises(NotImplementedError):
            fn(model, shape, cond_fn_with_grad=True)
        with pytest.raises(NotImplementedError):
            fn(model, shape, randomize_class=True)
        for bad in (0, 3, -1):
            with pytest.raises(ValueError):
                fn(model, shape, order=bad)
        for bad in (2.0, 1.5, "2", True, None):
            with pytest.raises(TypeError):
                fn(model, shape, order=bad)
        with pytest.raises(ValueError, match="noise_tape"):
            fn(model, shape, noise_tape=torch.zeros((6,) + shape))
    with pytest.raises(NotImplementedError):
        loop(model, shape, dump_steps=[1])
    with pytest.raises(NotImplementedError):
        loop(model, shape, const_noise=True)


def test_c_abi_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    lib.b200mdm_last_error.restype = ctypes.c_char_p
    buf = ctypes.c_void_p(16)               # never dereferenced: every call below fails its argument checks first

    def err(code, want, text):
        assert code == want, code
        assert text in lib.b200mdm_last_error(), lib.b200mdm_last_error()
    loop = lib.b200mdm_dpm_loop_range
    for order in (0, 3, -1):
        err(loop(None, order, 5, 6, buf, buf, 0, 1, None), _lib.EINVAL, b"order")
    err(loop(None, 2, 5, 6, buf, buf, _lib.FLAG_PHILOX_NOISE, 1, None), _lib.EINVAL, b"flag")
    err(loop(None, 2, 5, 6, buf, buf, _lib.FLAG_CONST_NOISE, 1, None), _lib.EINVAL, b"flag")
    err(loop(None, 2, 5, 0, buf, buf, 0, 1, None), _lib.EINVAL, b"step range")
    err(loop(None, 2, 5, 6, buf, buf, _lib.FLAG_CLIP_DENOISED, 1, None), _lib.EINVAL, b"null engine")
    rows = np.zeros((6, _lib.SCHED_DPM_STRIDE), dtype=np.float32)
    err(lib.b200mdm_set_schedule_dpm(None, 6, rows.ctypes.data_as(ctypes.c_void_p)), _lib.EINVAL, b"bad argument")
    err(lib.b200mdm_dpm_pred_xstart(None, buf, None), _lib.EINVAL, b"null")
    hook = lib.b200mdm_test_out_dpm
    good = [buf, None, buf, buf, buf, buf, 3, 1, 2, 0, None, None, buf, buf, 2, 263, 24, 512, 1, 1, None]

    def with_(**over):
        names = ["h", "scale", "w", "b", "x", "row", "index", "step", "order", "flags", "mask", "motion", "hist", "out",
                 "B", "JF", "T", "d", "s_off", "halves", "stream"]
        a = list(good)
        for k, v in over.items():
            a[names.index(k)] = v
        return hook(*a)
    for over in (dict(order=0), dict(order=3), dict(index=-1), dict(step=-1), dict(flags=_lib.FLAG_CONST_NOISE),
                 dict(row=None), dict(hist=None), dict(out=None), dict(x=None), dict(mask=buf), dict(halves=2),
                 dict(d=100), dict(B=0)):
        err(with_(**over), _lib.EINVAL, b"bad argument")
