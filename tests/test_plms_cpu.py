"""CPU: pseudo linear multistep sampling (diffusion/gaussian_diffusion.py:992-1187 of the reference) -- the fp32 oracle
against the reference's golden outputs, argument checks of the Python API and of the C ABI that run before any device
work, and the schedule columns the PLMS epilogue reads."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from conftest import default_args
from oracle import gen_golden_plms as gp
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ref_harness as rh
from oracle import schedule_oracle as so


def _enc_oracle_cases():
    c = gp.ENC
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    tmap = list(range(c["steps"]))
    inp, shape, imask, motion = gp.enc_inputs()
    xT = inp["tape"][0]
    cfg = po.enc_denoiser(W, tmap, inp["text_embed"], inp["scale"], inp["lengths"])
    bare = po.enc_denoiser(W, tmap, inp["text_embed"], None, inp["lengths"])
    steps = []
    out = {"enc_o2": po.plms_loop(cfg, tabs, xT, 2), "enc_o3": po.plms_loop(cfg, tabs, xT, 3)}
    po.plms_loop(cfg, tabs, xT, 4, collect=steps)
    out["enc_o4_steps"] = torch.stack(steps)
    out["enc_o2_clip"] = po.plms_loop(cfg, tabs, xT, 2, clip_denoised=True)
    out["enc_o2_inpaint"] = po.plms_loop(cfg, tabs, xT, 2, inpaint=(imask, motion))
    out["enc_o2_skip5"] = po.plms_loop(cfg, tabs, xT, 2, skip_timesteps=5)
    out["enc_o2_noguide"] = po.plms_loop(bare, tabs, xT, 2)
    return out


def test_oracle_vs_golden(golden):
    g = golden("plms_small.npz")
    for name, o in _enc_oracle_cases().items():
        np.testing.assert_allclose(o.numpy(), g[name], rtol=1e-4, atol=1e-4, err_msg=name)
    c = gp.DIP
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                      seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    inp, enc, tmask, prefix = gp.dip_inputs()
    f = po.dec_denoiser(W, list(range(c["steps"])), enc, tmask, prefix, inp["scale"], inp["lengths"])
    np.testing.assert_allclose(po.plms_loop(f, tabs, inp["tape"][0], 2).numpy(), g["dip_o2"], rtol=1e-4, atol=1e-4)


@pytest.mark.skipif(not rh.available(), reason="reference tree not present")
def test_golden_reproduces_from_generator(golden, tmp_path, monkeypatch):
    g = golden("plms_small.npz")
    monkeypatch.setattr(gp, "OUT", str(tmp_path))
    new = gp.gen_plms_small()
    assert set(new) == set(g.files)
    for k in g.files:
        if k != "meta":
            np.testing.assert_allclose(new[k], g[k], rtol=1e-6, atol=1e-6, err_msg=k)


def _diffusion():
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=6),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    return model, diffusion


def test_order_checked_before_any_device_work(monkeypatch):
    model, diffusion = _diffusion()

    def no_engine(*a, **k):
        raise AssertionError("the engine was reached")
    monkeypatch.setattr(type(diffusion), "_prepare", no_engine)
    shape = (2, 263, 1, 24)
    t = torch.full((2,), 3, dtype=torch.long)
    x = torch.zeros(shape)
    for order in (0, 5, 2.5, "2"):
        with pytest.raises(ValueError):
            diffusion.plms_sample_loop(model, shape, order=order)
        with pytest.raises(ValueError):
            next(diffusion.plms_sample_loop_progressive(model, shape, order=order))
        with pytest.raises(ValueError):
            diffusion.plms_sample(model, x, t, order=order)
    with pytest.raises(TypeError):
        diffusion.plms_sample_loop(model, shape, order=1)
    with pytest.raises(TypeError):
        next(diffusion.plms_sample_loop_progressive(model, shape, order=1))
    with pytest.raises(TypeError):
        diffusion.plms_sample(model, x, t, order=1)
    with pytest.raises(ValueError):
        diffusion.plms_sample_loop(model, shape, noise_tape=torch.zeros((6,) + shape))
    with pytest.raises(NotImplementedError):
        diffusion.plms_sample_loop(model, shape, cond_fn=lambda *a: 0)
    with pytest.raises(NotImplementedError):
        diffusion.plms_sample(model, x, t, denoised_fn=lambda v: v)


def test_c_abi_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    lib.b200mdm_last_error.restype = ctypes.c_char_p
    buf = ctypes.c_void_p(16)               # never dereferenced: every call below fails its argument checks first

    def err(code, text):
        assert code == _lib.EINVAL, code
        assert text in lib.b200mdm_last_error(), lib.b200mdm_last_error()
    loop = lib.b200mdm_plms_loop_range
    err(loop(None, 0, 5, 6, buf, buf, 0, 1, None), b"order 0")
    err(loop(None, 5, 5, 6, buf, buf, 0, 1, None), b"order 5")
    err(loop(None, 2, 5, 6, buf, buf, _lib.FLAG_PHILOX_NOISE, 1, None), b"flag")
    err(loop(None, 1, 5, 6, buf, buf, 0, 1, None), b"order 1")
    err(loop(None, 2, 5, 0, buf, buf, 0, 1, None), b"step range")
    err(loop(None, 2, 5, 6, buf, buf, 0, 1, None), b"null engine")
    step = lib.b200mdm_plms_step
    old = (ctypes.c_void_p * 3)(16, None, 16)
    err(step(None, 3, 0, buf, old, 1, 0, buf, None, None, None), b"order 0")
    err(step(None, 3, 2, buf, old, 1, _lib.FLAG_CONST_NOISE, buf, None, None, None), b"flag")
    err(step(None, 3, 2, buf, None, 2, 0, buf, None, None, None), b"history")
    err(step(None, 3, 2, buf, old, -1, 0, buf, None, None, None), b"history")
    err(step(None, 3, 1, buf, None, 0, 0, buf, None, None, None), b"order 1")      # no history array: old_out None
    err(step(None, 3, 1, buf, old, 0, 0, buf, None, None, None), b"null engine")   # an empty history is valid
    err(step(None, 3, 2, None, old, 1, 0, buf, None, None, None), b"null tensor")
    err(step(None, 3, 2, buf, old, 1, 0, None, None, None, None), b"null tensor")
    err(step(None, 3, 4, buf, old, 3, 0, buf, None, None, None), b"null eps history entry 1")
    err(step(None, 3, 2, buf, old, 1, 0, buf, None, None, None), b"null engine")


def test_schedule_columns_are_sqrt_abp_and_sqrt_one_minus_abp():
    """The PLMS epilogue reads sqrt(abp) and sqrt(1 - abp) (gaussian_diffusion.py:1045,1049,1066) from columns 5 and 6
    of the eta = 0 table: with sigma exactly 0, 1 - abp - sigma^2 is 1 - abp, bit for bit.  The fp32 square root is the
    correctly rounded one (the fp64 root rounded to fp32 is exact for sqrt), as on the GPU."""
    def sqrt32(v):
        return np.sqrt(v.astype(np.float64)).astype(np.float32)
    for n in (6, 50, 1000):
        _, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=n),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
        rows = diffusion.schedule_rows(0.0)
        abp = diffusion.alphas_cumprod_prev.astype(np.float32)          # _extract_into_tensor's fp32 values
        assert np.array_equal(rows[:, 5], sqrt32(abp)), n
        assert np.array_equal(rows[:, 6], sqrt32(np.float32(1) - abp)), n
        assert not rows[:, 7].any()
