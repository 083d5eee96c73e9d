"""CPU: joint-position control (JointControlSampleModel, b200mdm_set_joint_guidance; DESIGN.md "Joint-position control").

  * the fp64 oracle's gradient (autograd through oracle/ric_oracle.py) against central finite differences, for
    HumanML3D and KIT at T = 1, 2, 60; the kernel's written-out adjoint (guide_manual) against autograd;
  * a zero step and all-zero weights leave x0 as it was;
  * every refusal of the wrapper and the samplers that needs no GPU; the C ABI's argument checks, which run before any
    CUDA call; the new symbols in the header and _lib.SYMBOLS; shard_model_kwargs slices the two keys."""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import ROOT, default_args
from oracle import joint_control_oracle as jo


def _case(D, T, seed, B=2, density=0.4):
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    x0 = torch.randn(B, D, T, generator=g, dtype=torch.float64)
    target = torch.randn(B, J, 3, T, generator=g, dtype=torch.float64)
    weight = (torch.rand(B, J, T, generator=g) < density).double() * (0.5 + torch.rand(B, J, T, generator=g, dtype=torch.float64))
    weight[0, 0] = 1.0                                                   # the root on every frame of sample 0
    return x0, mean, std, target, weight


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [1, 2, 60])
def test_gradient_against_finite_differences(D, T):
    x0, mean, std, target, weight = _case(D, T, seed=D + T)
    x = x0.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(jo.loss(x, mean, std, target, weight).sum(), x)
    R = jo.ric_features(jo.n_joints(D))
    assert torch.equal(g[:, R:], torch.zeros_like(g[:, R:]))            # only the ric features have a gradient
    gen = torch.Generator().manual_seed(T)
    picks = torch.randint(0, 2 * R * T, (min(150, 2 * R * T),), generator=gen)
    h = 1e-6
    for k in picks.tolist():
        b, f, t = k // (R * T), (k // T) % R, k % T
        xp, xm = x0.clone(), x0.clone()
        xp[b, f, t] += h
        xm[b, f, t] -= h
        fd = (jo.loss(xp, mean, std, target, weight)[b] - jo.loss(xm, mean, std, target, weight)[b]) / (2 * h)
        assert abs(float(fd) - float(g[b, f, t])) <= 1e-6 * (1 + abs(float(fd))), (b, f, t, float(fd), float(g[b, f, t]))
    G2, g2 = jo.grad_manual(x0, mean, std, target, weight)
    assert torch.allclose(g2, g, rtol=1e-10, atol=1e-10 * float(g.abs().max() + 1))
    assert torch.allclose(G2, jo.loss(x0, mean, std, target, weight), rtol=1e-12)


@pytest.mark.parametrize("D", [263, 251])
def test_mutants_change_the_result(D):
    x0, mean, std, target, weight = _case(D, 60, seed=5)
    step = jo.step_bound(std, weight, 4.0, 60)
    want, _ = jo.guide(x0, mean, std, target, weight, step, 3)
    got, _ = jo.guide_manual(x0, mean, std, target, weight, step, 3)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12)
    for m in ("sign", "no_yaw", "vel_shift", "no_std"):
        mut, _ = jo.guide_manual(x0, mean, std, target, weight, step, 3, mutant=m)
        assert float((mut - want).abs().max()) > 1e-6, m


def test_zero_step_and_zero_weights_are_the_identity():
    x0, mean, std, target, weight = _case(263, 24, seed=2)
    out, losses = jo.guide(x0, mean, std, target, weight, 0.0, 3)
    assert torch.equal(out, x0) and torch.equal(losses[0], losses[-1])
    out, losses = jo.guide(x0, mean, std, target, torch.zeros_like(weight), 0.5, 3)
    assert torch.equal(out, x0) and float(losses.abs().max()) == 0.0
    target.masked_fill_((weight == 0)[:, :, None, :], float("nan"))      # a free joint's target is never read
    out, _ = jo.guide(x0, mean, std, target, weight, 1e-3, 2)
    assert bool(torch.isfinite(out).all())


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_wrapper_and_sampler_refusals():
    model, diffusion = _model()
    mean, std = jo.motion_stats(263)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4)
    assert jc.njoints == 263 and jc.cond_mask_prob == 0.1 and jc.n_iters == 4 and jc.n_joints == 22
    for bad in (dict(step_size=0.0), dict(step_size=float("nan")), dict(step_size=-1.0), dict(n_iters=0),
                dict(n_iters=10001), dict(n_iters=2.5), dict(mean=mean[:10])):
        kw = dict(model=cfg, mean=mean, std=std, step_size=1e-3, n_iters=4)
        kw.update(bad)
        with pytest.raises(ValueError):
            b200mdm.JointControlSampleModel(**kw)
    with pytest.raises(TypeError):
        b200mdm.JointControlSampleModel(SimpleNamespace(model=model), mean, std, 1e-3, 4)
    with pytest.raises(TypeError):
        b200mdm.HandshakeSampleModel(jc, 4)
    with pytest.raises(TypeError):
        b200mdm.JointControlSampleModel(b200mdm.HandshakeSampleModel(cfg, 4), mean, std, 1e-3, 4)
    a2m, _ = _model(dataset="humanact12", unconstrained=False)
    with pytest.raises(ValueError):
        b200mdm.JointControlSampleModel(a2m, mean, std, 1e-3, 4)
    dip, _ = _model(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    with pytest.raises(NotImplementedError):
        b200mdm.JointControlSampleModel(dip, mean, std, 1e-3, 4)
    B, T = 2, 24
    x = torch.zeros(B, 263, 1, T)
    t = torch.zeros(B, dtype=torch.long)
    y = {"text_embed": torch.zeros(1, B, 512), "scale": torch.ones(B), "joint_target": torch.zeros(B, 22, 3, T),
         "joint_weight": torch.ones(B, 22, T)}
    kw = {"y": y}
    for call in (lambda: diffusion.plms_sample_loop(jc, x.shape, model_kwargs=kw),
                 lambda: next(diffusion.plms_sample_loop_progressive(jc, x.shape, model_kwargs=kw)),
                 lambda: diffusion.plms_sample(jc, x, t, model_kwargs=kw),
                 lambda: diffusion.dpm_solver_sample_loop(jc, x.shape, model_kwargs=kw),
                 lambda: next(diffusion.dpm_solver_sample_loop_progressive(jc, x.shape, model_kwargs=kw)),
                 lambda: diffusion.ddim_reverse_sample_loop(jc, x, model_kwargs=kw),
                 lambda: diffusion.ddim_reverse_sample(jc, x, t, model_kwargs=kw),
                 lambda: next(diffusion.ddim_reverse_sample_loop_progressive(jc, x, model_kwargs=kw)),
                 lambda: diffusion.calc_bpd_loop(jc, x, model_kwargs=kw),
                 lambda: diffusion.p_mean_variance(jc, x, t, model_kwargs=kw),
                 lambda: b200mdm.AutoRegressiveSampler(SimpleNamespace(pred_len=12, context_len=12), diffusion.p_sample_loop)
                 .sample(jc, x.shape, model_kwargs={"y": dict(y, prefix=torch.zeros(B, 263, 1, 12))})):
        with pytest.raises(NotImplementedError):
            call()
    with pytest.raises(TypeError):
        b200mdm.refine_transitions(diffusion.p_sample_loop, jc, x, kw, 2, 2, 1)
    # y: missing or mis-shaped keys, bad weights; never mutated
    snapshot = dict(y)
    for bad in ({"joint_target": None}, {"joint_weight": None}, {"joint_target": torch.zeros(B, 21, 3, T)},
                {"joint_weight": torch.zeros(B, 22, T + 1)}, {"joint_weight": -torch.ones(B, 22, T)},
                {"joint_weight": torch.ones(B, 22, T, dtype=torch.long)},
                {"joint_target": torch.full((B, 22, 3, T), float("inf"))}):
        yy = {k: v for k, v in dict(y, **bad).items() if v is not None}
        for call in (lambda: diffusion.p_sample_loop(jc, x.shape, model_kwargs={"y": yy}),
                     lambda: diffusion.ddim_sample(jc, x, t, model_kwargs={"y": yy})):
            with pytest.raises(ValueError):
                call()
    assert y.keys() == snapshot.keys() and all(y[k] is snapshot[k] for k in y)
    c, w = jc.targets(dict(y, joint_weight=torch.ones(B, 22, T, dtype=torch.bool)), x.shape)
    assert w.dtype == torch.float32 and float(w.min()) == 1.0 and c.shape == (B, 22, 3, T)


def test_shard_model_kwargs_slices_the_joint_keys():
    y = {"joint_target": torch.arange(6 * 22 * 3 * 4.0).view(6, 22, 3, 4), "joint_weight": torch.rand(6, 22, 4),
         "text_embed": torch.zeros(1, 6, 512)}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(part["joint_target"], y["joint_target"][2:5]) and torch.equal(part["joint_weight"], y["joint_weight"][2:5])


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    assert lib.b200mdm_set_joint_guidance(None, buf, buf, buf, buf, ctypes.c_float(1e-3), 4, None) == _lib.EINVAL

    def hook(x0=buf, mean=buf, B=2, T=60, D=263, step=1e-3, iters=4, out=buf):
        return lib.b200mdm_test_joint_guidance(x0, mean, buf, buf, buf, B, T, D, ctypes.c_float(step), iters, out, None, None)
    for kw, msg in ((dict(x0=None), b"null"), (dict(out=None), b"null"), (dict(mean=None), b"null"),
                    (dict(step=0.0), b"step"), (dict(step=-1.0), b"step"), (dict(step=float("inf")), b"step"),
                    (dict(step=float("nan")), b"step"), (dict(iters=0), b"iterations"), (dict(iters=10001), b"iterations"),
                    (dict(D=264), b"D 264"), (dict(T=257), b"T"), (dict(T=0), b"T"), (dict(B=0), b"B")):
        assert hook(**kw) == _lib.EINVAL, kw
        assert msg in lib.b200mdm_last_error(), (kw, lib.b200mdm_last_error())


def test_symbols_in_header_and_lib():
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    for name in ("b200mdm_set_joint_guidance", "b200mdm_test_joint_guidance"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)
