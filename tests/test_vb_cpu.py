"""CPU: the variational bound (calc_bpd_loop) and p_mean_variance without a GPU.

  * the fp32 oracle (oracle/vb_oracle.py) against every case of tests/golden/vb_small.npz, which the unmodified
    reference's calc_bpd_loop produced (oracle/gen_golden_vb.py);
  * the bound table (GaussianDiffusion.schedule_vb_rows) against the fp64 formulas, for FIXED_SMALL and FIXED_LARGE,
    plain and respaced;
  * the engine-order reduction restatement against fp64 sums;
  * the argument checks that refuse before any engine work, and the C ABI's new symbols."""
import importlib
import os
import re

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import gen_golden_vb as gv
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so
from oracle import vb_oracle as vo

deo = importlib.import_module("oracle.dec_emb_oracle")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-3


def case_oracle(case):
    """(denoise(x, i), fp64 tables, x_start, noise tape, inpaint, var_type, clip) of a vb_small.npz case, for the oracle."""
    args, sdkw, _, guided = gv.args_of(case)
    inp, shape, extra = gv.inputs(case)
    sd = b200mdm.synthetic_state_dict(**sdkw)
    L = sdkw["num_layers"]
    sc = inp["scale"] if guided else None
    if case == "respaced":
        betas, tmap, _ = so.respaced(so.named_betas("cosine", gv.RESP["base_steps"]),
                                     so.space_timesteps(gv.RESP["base_steps"], gv.RESP["respacing"]))
    else:
        betas, tmap = so.named_betas("cosine", args.diffusion_steps), list(range(args.diffusion_steps))
    tabs = so.diffusion_tables(betas)
    if case == "a2m":
        W = mo.OracleWeights(sd, L)
        act = extra["action"]

        def f(x, i):
            return mo.denoise_enc(W, x, int(tmap[i]), None, inp["lengths"], True, False, act)
    elif case == "dip":
        W = mo.OracleWeights(sd, L, arch="trans_dec")
        enc, tmask = extra["text_embed"]
        f = po.dec_denoiser(W, tmap, enc, tmask, extra["prefix"], sc, inp["lengths"])
    elif case == "clip_dec":
        W = mo.OracleWeights(sd, L)
        f = deo.denoiser(W, tmap, inp["text_embed"], sc, inp["lengths"])
    else:
        W = mo.OracleWeights(sd, L)
        f = po.enc_denoiser(W, tmap, inp["text_embed"], sc, inp["lengths"])
    inpaint = (extra["inpainting_mask"], extra["inpainted_motion"]) if "inpainting_mask" in extra else None
    var = "large" if case == "enc_large" else "small"
    return f, tabs, inp["tape"][0], inp["tape"][1:], inpaint, var, case == "enc_clip_inpaint"


def golden_case(case):
    g = np.load(os.path.join(ROOT, "tests", "golden", "vb_small.npz"))
    return {k: torch.from_numpy(g["%s_%s" % (case, k)]) for k in gv.KEYS}


@pytest.mark.parametrize("case", gv.CASES)
def test_oracle_vs_golden(case):
    f, tabs, xs, tape, inpaint, var, clip = case_oracle(case)
    want = golden_case(case)
    with torch.no_grad():
        got = vo.vb_loop(f, tabs, xs, tape, clip, inpaint, var)
    for k in gv.KEYS:
        e = rel_err(got[k], want[k])
        print("%s %s: relative error vs the reference %.2e" % (case, k, e))
        assert got[k].shape == want[k].shape and e < RTOL, (case, k, e)
    assert torch.all(want["vb"] > 0)


def _diffusions():
    out = []
    for small in (True, False):
        var = gd.ModelVarType.FIXED_SMALL if small else gd.ModelVarType.FIXED_LARGE
        for steps, resp in ((8, None), (1000, None), (1000, "ddim10"), (50, None)):
            kw = dict(betas=gd.get_named_beta_schedule("cosine", steps), model_mean_type=gd.ModelMeanType.START_X,
                      model_var_type=var, loss_type=gd.LossType.MSE)
            out.append(rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(steps, resp), **kw) if resp
                       else gd.GaussianDiffusion(**kw))
    return out


def test_table_vs_fp64():
    for d in _diffusions():
        rows = d.schedule_vb_rows()
        assert rows.dtype == np.float32 and rows.shape == (d.num_timesteps, _lib.SCHED_VB_STRIDE)
        lvm = d._model_log_variance()
        plain = [d.posterior_mean_coef1, d.posterior_mean_coef2, d.posterior_log_variance_clipped, lvm,
                 d.sqrt_recip_alphas_cumprod, d.sqrt_recipm1_alphas_cumprod, d.sqrt_alphas_cumprod,
                 d.sqrt_one_minus_alphas_cumprod]
        for c, v in enumerate(plain):                      # the reference's fp32 tensors: fp64 rounded once
            assert np.array_equal(rows[:, c], np.asarray(v).astype(np.float32)), c
        lvt, lq = d.posterior_log_variance_clipped, d.log_one_minus_alphas_cumprod
        derived = {8: (-1.0 + lvm) - lvt + np.exp(lvt - lvm), 9: np.exp(-lvm), 10: np.exp(-0.5 * lvm),
                   11: (-1.0 - lq) + np.exp(lq)}
        for c, v in derived.items():
            # fp32 arithmetic on fp32 inputs: a few ulps of the operands' magnitude
            scale = {8: 2.0 + np.abs(lvt) + np.abs(lvm), 9: v, 10: v, 11: 1.0 + np.abs(lq) + np.exp(lq)}[c]
            err = np.abs(rows[:, c].astype(np.float64) - v) / scale
            assert err.max() < 8 * 2.0 ** -24 * (1 + np.abs(lvm).max()), (c, err.max())
        if d.model_var_type == gd.ModelVarType.FIXED_SMALL:
            assert np.array_equal(rows[:, 2], rows[:, 3])
            assert np.all(rows[:, 8] == np.float32(0.0)) or np.abs(rows[:, 8]).max() < 1e-6


def test_engine_order_sums():
    g = torch.Generator().manual_seed(3)
    for B, J, T in ((2, 263, 24), (3, 150, 60), (1, 263, 196)):
        e = torch.rand(B, J, T, generator=g, dtype=torch.float64).float()
        got = vo.engine_mean(e).double()
        want = e.double().mean(dim=(1, 2))
        # two-level fp32 summation of J*T non-negative terms: |err| <= (32 + J*T/256 + 8) u * sum
        assert torch.all((got - want).abs() <= (40 + J * T / 256) * 2.0 ** -24 * want), (got, want)
        assert not torch.equal(vo.engine_mean(e, drop_last_chunk=True), vo.engine_mean(e))


def test_argument_checks():
    d = gd.GaussianDiffusion(betas=gd.get_named_beta_schedule("cosine", 8), model_mean_type=gd.ModelMeanType.START_X,
                             model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    x = torch.zeros(2, 263, 1, 24)
    with pytest.raises(NotImplementedError):
        d.p_mean_variance(None, x, torch.tensor([3, 3]), denoised_fn=lambda z: z)
    with pytest.raises(AssertionError):
        d.p_mean_variance(None, x, torch.tensor([3, 2]))
    with pytest.raises(ValueError):
        d.calc_bpd_loop(None, x, noise_tape=torch.zeros(8, *x.shape), noise_seed=1)
    learned = gd.GaussianDiffusion(betas=gd.get_named_beta_schedule("cosine", 8), model_mean_type=gd.ModelMeanType.START_X,
                                   model_var_type=gd.ModelVarType.LEARNED_RANGE, loss_type=gd.LossType.MSE)
    with pytest.raises(NotImplementedError):
        learned.calc_bpd_loop(None, x)
    with pytest.raises(NotImplementedError):
        learned.p_mean_variance(None, x, torch.tensor([3, 3]))
    with pytest.raises(NotImplementedError):                  # training stays out of scope
        d.training_losses(None, x, torch.tensor([3, 3]))


def test_q_tables():
    d = gd.GaussianDiffusion(betas=gd.get_named_beta_schedule("cosine", 8), model_mean_type=gd.ModelMeanType.START_X,
                             model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    x, xt = torch.randn(2, 263, 1, 5), torch.randn(2, 263, 1, 5)
    t = torch.tensor([5, 2])
    m, v, lv = d.q_mean_variance(x, t)
    assert torch.equal(m, torch.tensor(np.float32(d.sqrt_alphas_cumprod[[5, 2]])).view(2, 1, 1, 1) * x)
    assert torch.equal(v[:, 0, 0, 0], torch.tensor((1.0 - d.alphas_cumprod[[5, 2]]).astype(np.float32)))
    assert torch.equal(lv[:, 0, 0, 0], torch.tensor(d.log_one_minus_alphas_cumprod[[5, 2]].astype(np.float32)))
    pm, pv, plv = d.q_posterior_mean_variance(x, xt, t)
    tabs = so.diffusion_tables(d.betas)
    for b, i in enumerate((5, 2)):
        want = mo.f32(tabs["posterior_mean_coef1"], i) * x[b] + mo.f32(tabs["posterior_mean_coef2"], i) * xt[b]
        assert torch.equal(pm[b], want)
        assert float(pv[b].flatten()[0]) == np.float32(d.posterior_variance[i])
        assert float(plv[b].flatten()[0]) == np.float32(d.posterior_log_variance_clipped[i])


def test_abi_symbols():
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    for name in ("b200mdm_set_schedule_vb", "b200mdm_vb_loop_range", "b200mdm_test_out_vb"):
        assert name in _lib.SYMBOLS
        assert re.search(r"\bint %s\(" % name, header), name
    assert "#define B200MDM_SCHED_VB_STRIDE 12" in header and _lib.SCHED_VB_STRIDE == 12
    lib = _lib.load()
    for name in ("b200mdm_set_schedule_vb", "b200mdm_vb_loop_range", "b200mdm_test_out_vb"):
        getattr(lib, name)
