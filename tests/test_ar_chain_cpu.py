"""CPU: DiP's autoregressive chain as engine loops, without a GPU -- which sample_fns AutoRegressiveSampler hands to the
engine (utils/sampler_util._chain_plan), the fp32 oracle chain against the unmodified reference's chain
(tests/golden/dip_ar_small.npz), and the C ABI's rejections before any CUDA call."""
import ctypes
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import respace as rs
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.utils.sampler_util import _chain_plan
from conftest import default_args, rel_err
from oracle import mdm_oracle as mo
from oracle import schedule_oracle as so

ga = importlib.import_module("oracle.gen_golden_ar_chain")

SHAPE = (2, 263, 1, 40)


def dip(**over):
    args = default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40,
                        **over)
    return b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))


def kw(**extra):
    return dict(model_kwargs={"y": {"prefix": torch.zeros(2, 263, 1, 20)}}, **extra)


def test_eligible_samplers():
    model, diffusion = dip()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    for fn, mode in ((diffusion.p_sample_loop, _lib.MODE_DDPM), (diffusion.ddim_sample_loop, _lib.MODE_DDIM),
                     (diffusion.dpm_solver_sample_loop, _lib.MODE_DPM)):
        for m in (model, cfg):
            plan = _chain_plan(fn, m, SHAPE, 5, kw())
            assert plan is not None and plan[0] is diffusion and plan[1] == mode
    spaced = rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(20, "4"), betas=gd.get_named_beta_schedule("cosine", 20),
                                model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL,
                                loss_type=gd.LossType.MSE)
    assert _chain_plan(spaced.ddim_sample_loop, cfg, SHAPE, 5, kw(eta=0.5))[2]["eta"] == 0.5
    assert _chain_plan(diffusion.dpm_solver_sample_loop, cfg, SHAPE, 5, kw(order=1))[2]["order"] == 1


def test_host_chain_for_everything_else():
    model, diffusion = dip()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    none = [
        (lambda *a, **k: diffusion.p_sample_loop(*a, **k), cfg, kw()),           # any other callable
        (diffusion.plms_sample_loop, cfg, kw()),
        (diffusion.p_sample_loop_progressive, cfg, kw()),
        (diffusion.p_sample_loop, cfg, kw(dump_steps=[1])),
        (diffusion.p_sample_loop, cfg, kw(const_noise=True)),
        (diffusion.p_sample_loop, cfg, kw(skip_timesteps=2)),
        (diffusion.p_sample_loop, cfg, kw(init_image=torch.zeros(SHAPE))),
        (diffusion.p_sample_loop, cfg, kw(denoised_fn=lambda x: x)),
        (diffusion.p_sample_loop, cfg, kw(cond_fn=lambda x, t: x)),
        (diffusion.p_sample_loop, cfg, kw(noise_fn=lambda b, k: None)),
        (diffusion.ddim_sample_loop, cfg, kw(noise_fn=None)),                  # no such keyword: the host chain's TypeError
        (diffusion.dpm_solver_sample_loop, cfg, kw(noise_fn=None)),
        (diffusion.p_sample_loop, cfg, kw(unknown_keyword=1)),
        (diffusion.p_sample_loop, cfg, kw(noise_seed=3, noise_tape=torch.zeros((5, 4) + SHAPE))),
        (diffusion.p_sample_loop, cfg, kw(noise_tape=torch.zeros((5, 3) + SHAPE))),          # not one row per step
        (diffusion.p_sample_loop, cfg, kw(noise=torch.zeros((4,) + SHAPE))),                 # fewer x_T than chunks
        (diffusion.dpm_solver_sample_loop, cfg, kw(order=3)),
        (diffusion.dpm_solver_sample_loop, cfg, kw(noise_tape=torch.zeros((5, 4) + SHAPE))),
        (diffusion.p_sample_loop, cfg, dict(model_kwargs={"y": {"prefix": torch.zeros(2, 263, 1, 20, dtype=torch.float64)}})),
    ]
    for fn, m, k in none:
        assert _chain_plan(fn, m, SHAPE, 5, k) is None
    enc, _ = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4), SimpleNamespace(dataset=SimpleNamespace()))
    assert _chain_plan(diffusion.p_sample_loop, enc, SHAPE, 5, kw()) is None                 # not a DiP model
    hs = b200mdm.HandshakeSampleModel(enc, 2)
    assert _chain_plan(diffusion.p_sample_loop, hs, SHAPE, 5, kw()) is None

    class Mine(gd.GaussianDiffusion):
        def p_sample_loop(self, *a, **k):
            return super().p_sample_loop(*a, **k)
    mine = Mine(betas=gd.get_named_beta_schedule("cosine", 4), model_mean_type=gd.ModelMeanType.START_X,
                model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    assert _chain_plan(mine.p_sample_loop, cfg, SHAPE, 5, kw()) is None                       # overridden by a subclass


def oracle_chain(case):
    """The fp32 oracle (mdm_oracle's DiP denoiser with CFG and its p_sample step) chained as the reference chains it:
    chunk c from the tape's x_T and eps of chunk c, conditioned on chunk c's prompts and the previous chunk's last
    context_len frames; the prefix in front with include_prefix; cropped at required_frames."""
    cfg = ga.CASES[case]
    inp = ga.inputs(case)
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=ga.L, cond_dim=768, seed=ga.WEIGHTS_SEED)
    W = mo.OracleWeights(sd, ga.L, arch="trans_dec")
    tabs = so.diffusion_tables(so.named_betas("cosine", ga.STEPS))
    prefix, pieces = inp["prefix"], []
    if cfg["include_prefix"]:
        pieces.append(prefix)
    for c in range(inp["x_T"].shape[0]):
        tape = [inp["x_T"][c]] + list(inp["eps"][c])
        x = mo.sample_loop_dec(W, tabs, list(range(ga.STEPS)), tape, inp["enc"][c], inp["pad"][c], prefix, inp["scale"],
                               inp["lengths"])
        pieces.append(x)
        prefix = x[..., -ga.CTX:]
    return torch.cat(pieces, -1)[..., :cfg["required"]]


@pytest.mark.parametrize("case", sorted(ga.CASES))
def test_oracle_chain_against_the_reference_fixture(golden, case):
    """tests/golden/dip_ar_small.npz: the unmodified reference's AutoRegressiveSampler (oracle/gen_golden_ar_chain.py) --
    chunk count, prefix hand-off, include_prefix offset and crop -- against the fp32 oracle chained the same way."""
    g = golden("dip_ar_small.npz")
    assert np.allclose(g[case + "_inputs_sum"], ga.inputs_sum(ga.inputs(case)), rtol=0, atol=0)   # the seeds regenerate
    ref = torch.from_numpy(g[case + "_sample"])
    assert ref.shape == (ga.B, 263, 1, ga.CASES[case]["required"])
    assert rel_err(oracle_chain(case), ref) < 1e-3


def test_c_abi_rejects_before_any_cuda_call():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    handle = ctypes.c_void_p(ctypes.addressof(buf))    # never dereferenced: the argument checks come first
    mask = (ctypes.c_uint8 * 16)()

    def setup(h=handle, n=5, pred=40, ctx=20, include=0, crop=196, enc=buf, m=mask):
        return lib.b200mdm_chain_setup(h, n, pred, ctx, include, crop, enc, m, None)
    assert setup(h=None) == _lib.EINVAL
    assert setup(n=0) == _lib.EINVAL and setup(n=-1) == _lib.EINVAL
    assert setup(ctx=0) == _lib.EINVAL and setup(ctx=41) == _lib.EINVAL and setup(pred=0) == _lib.EINVAL
    assert setup(crop=201) == _lib.EINVAL and b"crop" in lib.b200mdm_last_error()          # past the chain's 200 frames
    assert setup(crop=221, include=1) == _lib.EINVAL and setup(crop=0) == _lib.EINVAL
    assert setup(enc=None) == _lib.EINVAL and setup(m=None) == _lib.EINVAL

    def loop(h=handle, mode=_lib.MODE_DDPM, order=0, first=0, n=10, x_T=buf, tape=buf, out=buf, flags=0):
        return lib.b200mdm_chain_loop_range(h, mode, order, first, n, x_T, 0, tape, 16, out, flags, 1, None)
    assert loop(h=None) == _lib.EINVAL
    for mode in (_lib.MODE_X0, _lib.MODE_PLMS_AB, _lib.MODE_DDIM_REVERSE, _lib.MODE_VB, 9):
        assert loop(mode=mode) == _lib.EINVAL
    assert loop(order=1) == _lib.EINVAL
    assert loop(mode=_lib.MODE_DPM, order=0) == _lib.EINVAL and loop(mode=_lib.MODE_DPM, order=3) == _lib.EINVAL
    assert loop(flags=_lib.FLAG_CONST_NOISE) == _lib.EINVAL
    assert loop(tape=None) == _lib.EINVAL and b"PHILOX" in lib.b200mdm_last_error()
    assert loop(x_T=None) == _lib.EINVAL and loop(mode=_lib.MODE_DPM, order=2, x_T=None) == _lib.EINVAL
    assert loop(out=None) == _lib.EINVAL
    assert loop(n=0) == _lib.EINVAL and loop(first=-1) == _lib.EINVAL
