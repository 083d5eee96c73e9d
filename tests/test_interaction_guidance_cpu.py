"""CPU: the interaction terms of joint-position control (DESIGN.md "Joint-position control", "Several characters in
one scene"): the fp64 oracle's gradient against finite differences and its written-out adjoint against autograd, each
mutant against the bound on the hook cases (the fp32 rounding of the oracle standing in for the engine), the wrapper's
and the C ABI's argument checks, and the scene-aligned batch shards."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import default_args
import interaction_cases as ic
from oracle import foot_guidance_oracle as fo
from oracle import interaction_guidance_oracle as io
from oracle import joint_control_oracle as jo

HOOK_STEP = {2: 3e5, 8: 1e6}   # the hook cases' step, in units of 1 / L_GN (DESIGN.md: the bound is loose by ~1e5)


def _zero(x0):
    B, D, T = x0.shape
    J = jo.n_joints(D)
    return torch.zeros(B, J, 3, T, dtype=torch.float64), torch.zeros(B, J, T, dtype=torch.float64)


@pytest.mark.parametrize("D,C", [(263, 2), (251, 3)])
def test_gradient_against_finite_differences(D, C):
    T = 6
    for seed in range(64):   # a case whose live pairs keep >= 1e-3 m from every kink, some of them within the margin
        x0, mean, std, inter, lengths = ic.case(D, T, C, seed, spacing=0.6)
        if ic.kink_distance(x0, mean, std, inter, lengths) >= 1e-3:
            break
    else:
        raise AssertionError("no case keeps the live pairs 1e-3 m from the kinks")
    x0 = x0.double()
    target, weight = _zero(x0)
    kappa = torch.zeros(x0.shape[0], 4, T, dtype=torch.float64)
    scene = io.Scene()
    x = x0.clone().requires_grad_(True)
    G = io.loss(x, mean, std, target, weight, scene, inter, kappa, lengths)
    (g,) = torch.autograd.grad(G.sum(), x)
    assert float(G.sum()) > 0 and float(g.abs().max()) > 0
    gen = torch.Generator().manual_seed(seed)
    R = jo.ric_features(jo.n_joints(D))
    h = 1e-6
    for _ in range(24):
        b, f, t = (int(torch.randint(n, (1,), generator=gen)) for n in (x0.shape[0], R, T))
        xp, xm = x0.clone(), x0.clone()
        xp[b, f, t] += h
        xm[b, f, t] -= h
        fd = (io.loss(xp, mean, std, target, weight, scene, inter, kappa, lengths).sum()
              - io.loss(xm, mean, std, target, weight, scene, inter, kappa, lengths).sum()) / (2 * h)
        assert abs(float(fd) - float(g[b, f, t])) <= 1e-6 * max(1.0, abs(float(fd))), (b, f, t, float(fd), float(g[b, f, t]))
    # the written-out adjoint against autograd
    Gm, gm = io.grad_manual(x0, mean, std, target, weight, scene, inter, None, lengths, kappa=kappa)
    assert float((Gm - G.detach()).abs().max()) <= 1e-10 * float(G.abs().max())
    assert float((gm - g).abs().max()) <= 1e-10 * float(g.abs().max())


def test_grad_manual_with_every_term():
    D, T, C = 263, 20, 2
    x0, mean, std, inter, lengths = ic.case(D, T, C, 5, per_scene=False)
    x0 = x0.double()
    g = torch.Generator().manual_seed(3)
    J = jo.n_joints(D)
    target = torch.randn(x0.shape[0], J, 3, T, generator=g, dtype=torch.float64)
    weight = (torch.rand(x0.shape[0], J, T, generator=g) < 0.2).double()
    o, c = (-2.0, -1.5), 0.25
    z = o[1] + c * torch.arange(12, dtype=torch.float64)
    xx = o[0] + c * torch.arange(14, dtype=torch.float64)
    sdf = b200mdm.SceneGrid(0.3 + 0.8 * xx[None, :] - 0.5 * z[:, None], o, c)
    scene = io.Scene(3.0, 5.0, -0.2, 2.0, 0.3, sdf, None)
    kappa = fo._kappa(x0, mean, std, None, lengths)
    x = x0.clone().requires_grad_(True)
    G = io.loss(x, mean, std, target, weight, scene, inter, kappa, lengths)
    (ga,) = torch.autograd.grad(G.sum(), x)
    Gm, gm = io.grad_manual(x0, mean, std, target, weight, scene, inter, None, lengths, kappa=kappa)
    assert float((gm - ga).abs().max()) <= 1e-10 * float(ga.abs().max())
    assert float((Gm - G.detach()).abs().max()) <= 1e-10 * float(G.abs().max())


@pytest.mark.parametrize("D,C", [(263, 2), (251, 8)])
def test_mutants_miss_the_bound(D, C):
    T, K = 60, 10
    x0, mean, std, inter, lengths = ic.case(D, T, C, D + C)
    target, weight = _zero(x0)
    step = ic.step(x0, mean, std, inter) * HOOK_STEP[C]
    want, loss = io.guide(x0, mean, std, target, weight, step, K, io.Scene(), inter, None, lengths)
    assert bool((loss[1:] <= loss[:-1] * (1 + 1e-9)).all())
    got = want.float().double()                       # the fp32 oracle in place of the engine
    bnd = ic.bound(want, x0, K)
    assert float((got - want).abs().max()) <= bnd
    man, _ = io.guide_manual(x0, mean, std, target, weight, step, K, io.Scene(), inter, None, lengths)
    assert float((man - want).abs().max()) <= 1e-3 * bnd
    for m in io.MUTANTS:
        mut, _ = io.guide_manual(x0, mean, std, target, weight, step, K, io.Scene(), inter, None, lengths, mutant=m)
        miss = float((mut - got).abs().max()) / bnd
        print("D %d C %d: mutant %-15s misses the bound %.1f-fold" % (D, C, m, miss))
        assert miss >= 8.0, m


def _model():
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_wrapper_checks():
    model, diffusion = _model()
    mean, std = jo.motion_stats(263)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    JC = b200mdm.JointControlSampleModel
    jc = JC(cfg, mean, std, 1e-3, 4, characters=2, interaction_weight=2.0, interaction_margin=0.3)
    assert (jc.characters, jc.interaction_weight, jc.interaction_margin) == (2, 2.0, 0.3)
    for bad in (dict(characters=0), dict(characters=9), dict(characters=2.0), dict(characters=True),
                dict(characters=2, interaction_weight=-1.0), dict(characters=2, interaction_weight=float("nan")),
                dict(characters=2, interaction_margin=-0.1), dict(characters=2, interaction_margin=float("inf")),
                dict(interaction_weight=1.0)):
        with pytest.raises(ValueError):
            JC(cfg, mean, std, 1e-3, 4, **bad)
    B, T = 4, 24
    shape = (B, 263, 1, T)
    pl = torch.zeros(B, 3)
    pairs = torch.tensor([[0, 20, 1, 21]])
    good = dict(scene_placement=pl, interaction_pairs=pairs, interaction_reach=torch.tensor([0.1]),
                interaction_pair_weight=torch.ones(1, T))
    c, w = jc.targets({}, shape)                      # the joint keys are optional
    assert float(w.abs().max()) == 0.0
    out = jc.interaction(good, shape)
    assert torch.equal(out[0], pl) and out[1].tolist() == [[0, 20, 1, 21]]
    assert jc.interaction(dict(good, interaction_pair_weight=torch.ones(2, 1, T)), shape)[3].shape == (2, 1, T)
    assert jc.interaction({"scene_placement": pl}, shape)[1:] == (None, None, None)
    plain = JC(cfg, mean, std, 1e-3, 4, floor_weight=1.0)
    assert plain.interaction({}, shape) is None
    y0 = {"text_embed": torch.zeros(1, B, 512), "scale": torch.ones(B)}
    bads = [(jc, {}), (jc, dict(good, scene_placement=torch.zeros(B, 2))),
            (jc, dict(good, scene_placement=torch.full((B, 3), float("nan")))),
            (jc, dict(good, interaction_pairs=torch.tensor([[0, 20, 0, 21]]))),       # a == b
            (jc, dict(good, interaction_pairs=torch.tensor([[0, 22, 1, 21]]))),       # joint out of range
            (jc, dict(good, interaction_pairs=torch.tensor([[2, 20, 1, 21]]))),       # character out of range
            (jc, dict(good, interaction_pairs=torch.tensor([[-1, 20, 1, 21]]))),
            (jc, dict(good, interaction_pairs=torch.tensor([[0.0, 20, 1, 21]]))),
            (jc, dict(good, interaction_reach=torch.tensor([-0.1]))),
            (jc, dict(good, interaction_reach=torch.tensor([float("inf")]))),
            (jc, {k: v for k, v in good.items() if k != "interaction_reach"}),
            (jc, dict(good, interaction_pair_weight=-torch.ones(1, T))),
            (jc, dict(good, interaction_pair_weight=torch.ones(1, T + 1))),
            (jc, dict(good, interaction_pair_weight=torch.ones(3, 1, T))),
            (plain, good)]                                                               # keys without characters
    snapshot = dict(good)
    for wrapper, extra in bads:
        for call in (lambda: diffusion.p_sample_loop(wrapper, shape, model_kwargs={"y": dict(y0, **extra)}),
                     lambda: diffusion.ddim_sample(wrapper, torch.zeros(shape), torch.zeros(B, dtype=torch.long),
                                                   model_kwargs={"y": dict(y0, **extra)})):
            with pytest.raises(ValueError):
                call()
    jc3 = JC(cfg, mean, std, 1e-3, 4, characters=3)
    with pytest.raises(ValueError):                   # B % C != 0
        diffusion.p_sample_loop(jc3, shape, model_kwargs={"y": dict(y0, scene_placement=pl)})
    assert all(good[k] is snapshot[k] for k in good)
    with pytest.raises(NotImplementedError):          # the refusals are joint control's
        diffusion.plms_sample_loop(jc, shape, model_kwargs={"y": dict(y0, **good)})


def test_shards_follow_scenes():
    B, T, C = 6, 5, 3
    y = {"scene_placement": torch.rand(B, 3), "interaction_pair_weight": torch.rand(B // C, 2, T),
         "interaction_pairs": torch.tensor([[0, 1, 2, 3], [1, 0, 0, 0]]), "interaction_reach": torch.rand(2),
         "text_embed": torch.zeros(1, B, 512)}
    part = parallel.shard_model_kwargs({"y": y}, 3, 6, characters=C)["y"]
    assert torch.equal(part["scene_placement"], y["scene_placement"][3:6])
    assert torch.equal(part["interaction_pair_weight"], y["interaction_pair_weight"][1:2])
    assert part["interaction_pairs"] is y["interaction_pairs"] and part["interaction_reach"] is y["interaction_reach"]
    shared = dict(y, interaction_pair_weight=torch.rand(2, T))
    assert parallel.shard_model_kwargs({"y": shared}, 0, 3, characters=C)["y"]["interaction_pair_weight"] is \
        shared["interaction_pair_weight"]
    for lo, hi in ((0, 4), (1, 3), (2, 6)):
        with pytest.raises(ValueError):
            parallel.shard_model_kwargs({"y": y}, lo, hi, characters=C)


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    f = ctypes.c_float
    buf = (ctypes.c_float * 64)()
    assert lib.b200mdm_set_interaction_guidance(None, 2, f(1.0), f(0.3), buf, None, 0, None, None, 0, None) == _lib.EINVAL

    def hook(B=4, T=60, C=2, w=1.0, r=0.3, pl=buf, rows=((0, 20, 1, 21),), reach=(0.1,), pw=buf, stride=0):
        n = len(rows)
        pr = (ctypes.c_int32 * max(4 * n, 1))(*[v for row in rows for v in row])
        rc = (ctypes.c_float * max(n, 1))(*reach)
        return lib.b200mdm_test_interaction_guidance(buf, buf, buf, buf, buf, None, None, B, T, 263, f(1e-3), 4, f(0.0),
                                                     f(0.0), f(0.0), f(0.0), f(0.0), None, None, C, f(w), f(r), pl, pr, n,
                                                     rc, pw, stride, buf, None, None)
    for kw, msg in ((dict(C=1), b"characters"), (dict(C=9), b"characters"), (dict(B=6, C=4), b"whole number"),
                    (dict(w=-1.0), b"interaction weight"), (dict(r=float("nan")), b"interaction weight"),
                    (dict(pl=None), b"placement"), (dict(rows=((0, 20, 0, 21),)), b"reach row"),
                    (dict(rows=((0, 22, 1, 21),)), b"reach row"), (dict(rows=((2, 20, 1, 21),)), b"reach row"),
                    (dict(reach=(-0.5,)), b"reach[0]"), (dict(pw=None), b"null reach rows"),
                    (dict(stride=59), b"pair weight stride")):
        assert hook(**kw) == _lib.EINVAL, kw
        assert msg in lib.b200mdm_last_error(), (kw, lib.b200mdm_last_error())


def test_symbols_in_header_and_lib():
    import os
    header = open(os.path.join(os.path.dirname(ic.__file__), "..", "include", "b200mdm.h")).read()
    for name in ("b200mdm_set_interaction_guidance", "b200mdm_test_interaction_guidance"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)
