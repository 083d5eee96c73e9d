"""CPU: the foot-contact and floor terms of joint-position control (DESIGN.md "Joint-position control", "Foot contact
and floor").

  * the fp64 oracle's gradient (autograd through oracle/ric_oracle.py) against central finite differences, HumanML3D and
    KIT at T = 1, 2, 60 with lengths < T; the written-out adjoint (grad_manual) against autograd; each mutant misses;
  * the contact mask derived from the reference's own extract_features output (tests/golden/foot_contact.npz) equals
    its foot_detect result, and foot_detect on the fixture's positions pins the channel-to-joint map and the (t, t+1)
    pair convention;
  * zero weights leave x0 as it was;
  * the wrapper's argument checks, y never mutated; the C ABI's checks before any CUDA call; the new symbols."""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import ROOT, default_args
from oracle import foot_guidance_oracle as fo
from oracle import joint_control_oracle as jo

CW, FW, FH = 3.0, 5.0, 0.3


def _case(D, T, seed, B=2):
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    x0 = torch.randn(B, D, T, generator=g, dtype=torch.float64)
    target = torch.randn(B, J, 3, T, generator=g, dtype=torch.float64)
    weight = (torch.rand(B, J, T, generator=g) < 0.3).double()
    lengths = torch.tensor([T, max(1, T - 7)])
    return x0, mean, std, target, weight, lengths


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [1, 2, 60])
def test_gradient_against_finite_differences(D, T):
    x0, mean, std, target, weight, lengths = _case(D, T, seed=D + T)
    kappa = fo._kappa(x0, mean, std, None, lengths)
    x = x0.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(fo.loss(x, mean, std, target, weight, CW, FW, FH, kappa, lengths).sum(), x)
    R = jo.ric_features(jo.n_joints(D))
    assert torch.equal(g[:, R:], torch.zeros_like(g[:, R:]))
    picks = torch.randint(0, 2 * R * T, (min(150, 2 * R * T),), generator=torch.Generator().manual_seed(T))
    h = 1e-6
    for k in picks.tolist():
        b, f, t = k // (R * T), (k // T) % R, k % T
        xp, xm = x0.clone(), x0.clone()
        xp[b, f, t] += h
        xm[b, f, t] -= h
        fd = (fo.loss(xp, mean, std, target, weight, CW, FW, FH, kappa, lengths)[b] -
              fo.loss(xm, mean, std, target, weight, CW, FW, FH, kappa, lengths)[b]) / (2 * h)
        assert abs(float(fd) - float(g[b, f, t])) <= 1e-6 * (1 + abs(float(fd))), (b, f, t, float(fd), float(g[b, f, t]))
    G2, g2 = fo.grad_manual(x0, mean, std, target, weight, CW, FW, FH, None, lengths)
    assert torch.allclose(g2, g, rtol=1e-10, atol=1e-10 * float(g.abs().max() + 1))
    assert torch.allclose(G2, fo.loss(x0, mean, std, target, weight, CW, FW, FH, kappa, lengths), rtol=1e-12)


@pytest.mark.parametrize("D", [263, 251])
def test_mutants_change_the_result(D):
    x0, mean, std, target, weight, lengths = _case(D, 60, seed=5)
    step = fo.step_bound(std, weight, 4.0, 60, CW, FW)
    want, _ = fo.guide(x0, mean, std, target, weight, step, 3, CW, FW, FH, None, lengths)
    got, _ = fo.guide_manual(x0, mean, std, target, weight, step, 3, CW, FW, FH, None, lengths)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12)
    for m in fo.MUTANTS:
        mut, _ = fo.guide_manual(x0, mean, std, target, weight, step, 3, CW, FW, FH, None, lengths, mutant=m)
        assert float((mut - want).abs().max()) > 1e-6, m


def test_zero_weights_are_joint_control():
    x0, mean, std, target, weight, lengths = _case(263, 24, seed=2)
    a, la = fo.guide(x0, mean, std, target, weight, 1e-3, 3, 0.0, 0.0, FH, None, lengths)
    b, lb = jo.guide(x0, mean, std, target, weight, 1e-3, 3)
    assert torch.equal(a, b) and torch.equal(la, lb)
    out, losses = fo.guide(x0, mean, std, target, torch.zeros_like(weight), 0.5, 3, 0.0, 0.0)
    assert torch.equal(out, x0) and float(losses.abs().max()) == 0.0


@pytest.mark.parametrize("name,D", [("hml", 263), ("kit", 251)])
def test_contact_channels_match_the_reference_foot_detect(name, D):
    z = np.load(os.path.join(ROOT, "tests", "golden", "foot_contact.npz"))
    feats, contact, pos = z[name + "_features"], z[name + "_contact"], z[name + "_positions"]   # [T-1, D], [T-1, 4], [T, J, 3]
    assert feats.shape[1] == D and contact.shape[1] == 4 and 0 < contact.mean() < 1
    # the derived mask of the features (mean 0, std 1: x0 is the features) is the reference's foot_detect output
    T = pos.shape[0]
    x0 = torch.zeros(1, D, T, dtype=torch.float64)
    x0[0, :, :-1] = torch.from_numpy(feats.T)
    kappa = fo.derive_contact(x0, torch.zeros(D), torch.ones(D))[0]                     # [4, T]
    assert np.array_equal(kappa[:, :-1].numpy().T, contact) and float(kappa[:, -1].abs().max()) == 0
    # channel k, row t is foot f_k's step from frame t to t + 1 (threshold 0.002 on the squared displacement)
    f = list(fo.FOOT_JOINTS[jo.n_joints(D)])
    step = ((pos[1:, f] - pos[:-1, f]) ** 2).sum(-1) < float(z["thres"])
    assert np.array_equal(step.astype(np.float64), contact)
    swapped = step[:, [2, 3, 0, 1]]
    assert not np.array_equal(swapped.astype(np.float64), contact)
    late = ((pos[1:, f][1:] - pos[1:, f][:-1]) ** 2).sum(-1) < float(z["thres"])
    assert not np.array_equal(late.astype(np.float64), contact[:-1])


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_wrapper_checks():
    model, diffusion = _model()
    mean, std = jo.motion_stats(263)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, contact_weight=1.0, floor_weight=0.5, floor_height=0.1)
    assert jc.foot and jc.contact_weight == 1.0 and jc.floor_height == 0.1
    assert not b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4).foot
    for bad in (dict(contact_weight=-1.0), dict(floor_weight=float("nan")), dict(contact_weight=float("inf")),
                dict(floor_height=float("inf"))):
        with pytest.raises(ValueError):
            b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, **bad)
    B, T = 2, 24
    shape = (B, 263, 1, T)
    x = torch.zeros(shape)
    t = torch.zeros(B, dtype=torch.long)
    # without foot terms the joint keys stay required; with them they are optional
    plain = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, contact_weight=0.0, floor_weight=0.0)
    with pytest.raises(ValueError):
        plain.targets({}, shape)
    c, w = jc.targets({}, shape)
    assert c.shape == (B, 22, 3, T) and float(w.abs().max()) == 0.0
    y = {"text_embed": torch.zeros(1, B, 512), "scale": torch.ones(B), "foot_contact": torch.ones(B, 4, T)}
    snapshot = dict(y)
    for bad in (torch.ones(B, 4, T + 1), torch.ones(B, 2, T), -torch.ones(B, 4, T), torch.full((B, 4, T), float("nan")),
                torch.ones(B, 4, T, dtype=torch.long), np.ones((B, 4, T), dtype=np.float32)):
        yy = dict(y, foot_contact=bad)
        for call in (lambda: diffusion.p_sample_loop(jc, shape, model_kwargs={"y": yy}),
                     lambda: diffusion.ddim_sample(jc, x, t, model_kwargs={"y": yy})):
            with pytest.raises(ValueError):
                call()
    assert y.keys() == snapshot.keys() and all(y[k] is snapshot[k] for k in y)
    k = jc.foot_contact(dict(y, foot_contact=torch.ones(B, 4, T, dtype=torch.bool)), shape)
    assert k.dtype == torch.float32 and float(k.min()) == 1.0
    assert plain.foot_contact(y, shape) is None                                        # no foot terms: the key is unread
    # the refusals are joint control's
    with pytest.raises(NotImplementedError):
        diffusion.plms_sample_loop(jc, shape, model_kwargs={"y": y})
    with pytest.raises(TypeError):
        b200mdm.HandshakeSampleModel(jc, 4)


def test_shard_model_kwargs_slices_foot_contact():
    y = {"foot_contact": torch.rand(6, 4, 5), "text_embed": torch.zeros(1, 6, 512)}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(part["foot_contact"], y["foot_contact"][2:5])


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    assert lib.b200mdm_set_foot_guidance(None, ctypes.c_float(1.0), ctypes.c_float(0.0), ctypes.c_float(0.0), None, None,
                                         None) == _lib.EINVAL
    buf = (ctypes.c_float * 16)()
    ln = (ctypes.c_int64 * 2)(5, -1)

    def hook(x0=buf, B=2, T=60, D=263, step=1e-3, iters=4, cw=1.0, fw=1.0, fh=0.0, lengths=None, out=buf):
        return lib.b200mdm_test_foot_guidance(x0, buf, buf, buf, buf, None, lengths, B, T, D, ctypes.c_float(step), iters,
                                              ctypes.c_float(cw), ctypes.c_float(fw), ctypes.c_float(fh), out, None, None)
    for kw, msg in ((dict(x0=None), b"null"), (dict(out=None), b"null"), (dict(step=0.0), b"step"),
                    (dict(iters=0), b"iterations"), (dict(D=264), b"D 264"), (dict(T=257), b"T"), (dict(B=0), b"B"),
                    (dict(cw=-1.0), b"weights"), (dict(fw=float("nan")), b"weights"), (dict(cw=float("inf")), b"weights"),
                    (dict(fh=float("inf")), b"height"), (dict(lengths=ln), b"lengths[1]")):
        assert hook(**kw) == _lib.EINVAL, kw
        assert msg in lib.b200mdm_last_error(), (kw, lib.b200mdm_last_error())


def test_symbols_in_header_and_lib():
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    for name in ("b200mdm_set_foot_guidance", "b200mdm_test_foot_guidance"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)
