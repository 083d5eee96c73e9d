"""CPU: DDIM inversion (ddim_reverse_sample, diffusion/gaussian_diffusion.py:838-874 of the reference) -- the fp32 oracle
against the reference's golden outputs, the reverse table bit for bit, and the argument checks of the Python API and
of the C ABI that run before any device work."""
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
from oracle import gen_golden_reverse as gr
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ref_harness as rh
from oracle import reverse_oracle as ro
from oracle import schedule_oracle as so


def _oracle(denoise, tables, x, clip=False, inpaint=None):
    return ro.reverse_loop(denoise, tables, x, clip_denoised=clip, inpaint=inpaint)


def _check(name, got, g):
    np.testing.assert_allclose(got.numpy(), g["%s_sample" % name], rtol=1e-4, atol=1e-4, err_msg=name)


def test_oracle_vs_golden(golden):
    g = golden("reverse_small.npz")
    c = gr.ENC
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    inp, _, imask, motion = gr.enc_inputs()
    f = po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], inp["lengths"])
    _check("enc", _oracle(f, tabs, inp["tape"][0]), g)
    _check("enc_clip_inpaint", _oracle(f, tabs, inp["tape"][0], True, (imask, motion)), g)

    c = gr.DIP
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                      seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    inp, enc, tmask, prefix = gr.dip_inputs()
    f = po.dec_denoiser(W, list(range(c["steps"])), enc, tmask, prefix, inp["scale"], inp["lengths"])
    _check("dip", _oracle(f, tabs, inp["tape"][0]), g)

    c = gr.RESP
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    betas, tmap, _ = so.respaced(so.named_betas("cosine", c["base_steps"]), so.space_timesteps(c["base_steps"], c["respacing"]))
    inp = gr.resp_inputs()
    f = po.enc_denoiser(W, tmap, inp["text_embed"], None, inp["lengths"])
    _check("respaced", _oracle(f, so.diffusion_tables(betas), inp["tape"][0]), g)


@pytest.mark.skipif(not rh.available(), reason="reference tree not present")
def test_golden_reproduces_from_generator(golden, tmp_path, monkeypatch):
    g = golden("reverse_small.npz")
    monkeypatch.setattr(gr, "OUT", str(tmp_path))
    new = gr.gen_reverse_small()
    assert set(new) == set(g.files)
    for k in g.files:
        if k != "meta":
            np.testing.assert_allclose(new[k], g[k], rtol=1e-6, atol=1e-6, err_msg=k)


def test_schedule_next_rows_bit_identical_to_reference(golden):
    """The rows are the correctly rounded fp32 square roots of the reference's own fp32 operands abn and 1 - abn, bit
    for bit: what torch's sqrt gives on CUDA.  The fixture's th.sqrt values were computed by torch on the CPU, whose
    vectorised fp32 sqrt is not always correctly rounded; they are within one ulp (15 of 2120 values differ)."""
    g = golden("reverse_small.npz")
    _, d50 = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=50),
                                                SimpleNamespace(dataset=SimpleNamespace()))
    _, d1000 = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=1000),
                                                  SimpleNamespace(dataset=SimpleNamespace()))
    for key, diffusion in (("next_cos50", d50), ("next_cos1000", d1000), ("next_respaced", gr.respaced_diffusion(gd, rs))):
        rows = diffusion.schedule_next_rows()
        ops = g[key + "_operands"]
        assert rows.dtype == np.float32 and rows.shape == ops.shape == (diffusion.num_timesteps, _lib.SCHED_NEXT_STRIDE)
        assert np.array_equal(rows, np.sqrt(ops.astype(np.float64)).astype(np.float32)), key
        ulp = np.abs(rows.view(np.int32).astype(np.int64) - g[key].view(np.int32))
        assert ulp.max() <= 1, key
        assert rows[-1].tolist() == [0.0, 1.0]


def test_arguments_checked_before_any_device_work(monkeypatch):
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=6),
                                                          SimpleNamespace(dataset=SimpleNamespace()))

    def no_engine(*a, **k):
        raise AssertionError("the engine was reached")
    monkeypatch.setattr(type(diffusion), "_prepare", no_engine)
    x = torch.zeros((2, 263, 1, 24))
    t = torch.full((2,), 3, dtype=torch.long)
    with pytest.raises(AssertionError, match="Reverse ODE only for deterministic path"):
        diffusion.ddim_reverse_sample(model, x, t, eta=0.5)
    with pytest.raises(NotImplementedError):
        diffusion.ddim_reverse_sample(model, x, t, denoised_fn=lambda v: v)
    for first, n in ((-1, None), (6, None), (0, 0), (0, 7), (4, 3), (1.0, None), (0, 2.5), (True, 1)):
        with pytest.raises(ValueError):
            diffusion.ddim_reverse_sample_loop(model, x, first_index=first, n_steps=n)
        with pytest.raises(ValueError):
            next(diffusion.ddim_reverse_sample_loop_progressive(model, x, first_index=first, n_steps=n))


def test_c_abi_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    lib.b200mdm_last_error.restype = ctypes.c_char_p
    buf = ctypes.c_void_p(16)               # never dereferenced: every call below fails its argument checks first

    def err(code, want, text):
        assert code == want, code
        assert text in lib.b200mdm_last_error(), lib.b200mdm_last_error()
    loop = lib.b200mdm_ddim_reverse_loop_range
    err(loop(None, 0, 6, buf, buf, _lib.FLAG_PHILOX_NOISE, 1, None), _lib.EINVAL, b"flag")
    err(loop(None, 0, 6, buf, buf, _lib.FLAG_CONST_NOISE, 1, None), _lib.EINVAL, b"flag")
    err(loop(None, 0, 0, buf, buf, 0, 1, None), _lib.EINVAL, b"step range")
    err(loop(None, -1, 2, buf, buf, 0, 1, None), _lib.EINVAL, b"step range")
    err(loop(None, 0, 6, buf, buf, _lib.FLAG_CLIP_DENOISED, 1, None), _lib.EINVAL, b"null engine")
    nxt = lib.b200mdm_set_schedule_next
    rows = np.zeros((6, 2), dtype=np.float32)
    err(nxt(None, 6, rows.ctypes.data_as(ctypes.c_void_p)), _lib.EINVAL, b"bad argument")
    err(lib.b200mdm_sample_step(None, _lib.MODE_DDIM_REVERSE, 0, buf, None, 0, buf, None, None), _lib.EINVAL,
        b"null engine")
