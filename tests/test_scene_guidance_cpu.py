"""CPU: the scene terms of joint-position control (DESIGN.md "Joint-position control", "Scene: obstacles and uneven
ground").

  * the fp64 oracle's gradient (autograd through oracle/ric_oracle.py) against central finite differences, HumanML3D and
    KIT at T = 1, 2, 60 with lengths < T, on curved grids placed so that no joint the terms act on lies within 1e-3 cell
    of a grid line (where the bilinear gradient jumps); the written-out adjoint (grad_manual) against autograd to 1e-10;
    each mutant misses;
  * no scene term is the foot-guidance oracle; SceneGrid.from_shapes / shape_sdf against closed forms;
  * SceneGrid's and the wrapper's argument checks, y never mutated; sharding of per-sample grids; the C ABI's checks
    before any CUDA call; the new symbols."""
import ctypes
import math
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
from oracle import scene_guidance_oracle as so
import scene_cases as sc

CW, FW, FH, OW, R = sc.CW, sc.FW, sc.FH, sc.OW, sc.R
curved_case, planar_case = sc.curved_case, sc.planar_case


def _terms(sdf, terrain):
    return (CW, FW, FH, OW, R, sdf, terrain)


@pytest.mark.parametrize("D", [263, 251])
@pytest.mark.parametrize("T", [1, 2, 60])
def test_gradient_against_finite_differences(D, T):
    x0, mean, std, target, weight, lengths, sdf, terrain, n_o, n_f = curved_case(D, T, seed=D + T)
    assert n_o > 0 and n_f > 0
    kappa = fo._kappa(x0, mean, std, None, lengths)
    args = (target, weight, CW, FW, FH, OW, R, sdf, terrain, kappa, lengths)
    x = x0.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(so.loss(x, mean, std, *args).sum(), x)
    Rf = jo.ric_features(jo.n_joints(D))
    assert torch.equal(g[:, Rf:], torch.zeros_like(g[:, Rf:]))
    picks = torch.randint(0, 2 * Rf * T, (min(150, 2 * Rf * T),), generator=torch.Generator().manual_seed(T))
    h = 1e-6
    for k in picks.tolist():
        b, f, t = k // (Rf * T), (k // T) % Rf, k % T
        xp, xm = x0.clone(), x0.clone()
        xp[b, f, t] += h
        xm[b, f, t] -= h
        fd = (so.loss(xp, mean, std, *args)[b] - so.loss(xm, mean, std, *args)[b]) / (2 * h)
        assert abs(float(fd) - float(g[b, f, t])) <= 1e-6 * (1 + abs(float(fd))), (b, f, t, float(fd), float(g[b, f, t]))
    G2, g2 = so.grad_manual(x0, mean, std, target, weight, *_terms(sdf, terrain), None, lengths)
    assert torch.allclose(g2, g, rtol=1e-10, atol=1e-10 * float(g.abs().max() + 1))
    assert torch.allclose(G2, so.loss(x0, mean, std, *args), rtol=1e-12)


@pytest.mark.parametrize("D", [263, 251])
def test_mutants_change_the_result(D):
    x0, mean, std, target, weight, lengths, sdf, terrain = planar_case(D, 60, seed=5)
    step = so.step_bound(std, weight, 6.0, 60, 0.0, FW, OW, sdf, terrain)
    terms = (0.0, FW, FH, OW, R, sdf, terrain, None, lengths)
    want, _ = so.guide(x0, mean, std, target, weight, step, 3, *terms)
    got, _ = so.guide_manual(x0, mean, std, target, weight, step, 3, *terms)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12)
    for m in so.MUTANTS:
        mut, _ = so.guide_manual(x0, mean, std, target, weight, step, 3, *terms, mutant=m)
        assert float((mut - want).abs().max()) > 1e-6, m


def test_no_scene_is_foot_guidance():
    x0, mean, std, target, weight, lengths, sdf, terrain = planar_case(263, 24, seed=2)
    weight = (torch.rand(weight.shape, generator=torch.Generator().manual_seed(3)) < 0.3).double()
    a, la = so.guide(x0, mean, std, target, weight, 1e-3, 3, CW, FW, FH, 0.0, R, None, None, None, lengths)
    b, lb = fo.guide(x0, mean, std, target, weight, 1e-3, 3, CW, FW, FH, None, lengths)
    assert torch.allclose(a, b, rtol=1e-12, atol=1e-14) and torch.allclose(la, lb, rtol=1e-12)
    # an all-zero terrain is the flat floor; an SDF at least r everywhere is no obstacle
    flat = b200mdm.SceneGrid(torch.zeros(5, 6), (0.0, 0.0), 1.0)
    far = b200mdm.SceneGrid(torch.full((5, 6), R + 0.5), (0.0, 0.0), 1.0)
    c, lc = so.guide(x0, mean, std, target, weight, 1e-3, 3, CW, FW, FH, OW, R, far, flat, None, lengths)
    assert torch.allclose(c, b, rtol=1e-12, atol=1e-14) and torch.allclose(lc, lb, rtol=1e-12)


def test_shape_sdf_against_closed_forms():
    disc, box = (1.0, -2.0, 0.5), (2.0, 1.0, 4.0, 2.0)
    # disc centre and rim, box corner, centre, inside near an edge, beside an edge, past a corner
    pts = {(1.0, -2.0): -0.5, (1.0, -1.0): 0.5, (4.0, 2.0): 0.0, (3.0, 1.5): -0.5, (3.5, 1.2): -0.2, (5.0, 1.5): 1.0,
           (3.0, 0.0): 1.0, (5.0, 3.0): math.sqrt(2), (1.5, 1.0): 0.5}
    for (x, z), want in pts.items():
        d = b200mdm.shape_sdf(np.array([x]), np.array([z]), discs=[disc], boxes=[box])[0]
        assert abs(d - want) < 1e-12, (x, z, d, want)
    # each shape alone, on its own
    assert abs(b200mdm.shape_sdf(4.0, 2.0, boxes=[box]) - 0.0) < 1e-12
    assert abs(b200mdm.shape_sdf(4.5, 2.5, boxes=[box]) - math.sqrt(0.5)) < 1e-12
    assert abs(b200mdm.shape_sdf(1.3, -2.4, discs=[disc]) - (0.5 - 0.5)) < 1e-12
    # the grid holds the fp32 rounding of shape_sdf at its nodes, row i at z0 + i c, column k at x0 + k c
    g = b200mdm.SceneGrid.from_shapes((7, 9), (-1.0, -3.0), 0.5, discs=[disc], boxes=[box])
    assert g.shape == (7, 9) and not g.per_sample and g.values.dtype == torch.float32
    for i, k in ((0, 0), (2, 4), (6, 8), (5, 1)):
        want = b200mdm.shape_sdf(-1.0 + 0.5 * k, -3.0 + 0.5 * i, discs=[disc], boxes=[box])
        assert float(g.values[i, k]) == float(np.float32(want))
    # union: the smallest signed distance; sampling a grid node gives its value, between nodes the bilinear blend
    x, z = torch.tensor([[-1.0 + 0.5 * 4, -1.0 + 0.5 * 4.25]], dtype=torch.float64), torch.tensor([[-3.0 + 0.5 * 2] * 2],
                                                                                                    dtype=torch.float64)
    val, dx, dz = so.sample(g, x, z)
    assert float(val[0, 0]) == float(g.values[2, 4])
    assert abs(float(val[0, 1]) - (0.75 * float(g.values[2, 4]) + 0.25 * float(g.values[2, 5]))) < 1e-12
    assert abs(float(dx[0, 1]) - (float(g.values[2, 5]) - float(g.values[2, 4])) / 0.5) < 1e-12
    # outside the grid the value clamps and the gradient along the clamped axis is 0
    val, dx, dz = so.sample(g, torch.tensor([[-5.0]], dtype=torch.float64), torch.tensor([[-3.0 + 0.5 * 2.5]], dtype=torch.float64))
    assert float(dx[0, 0]) == 0.0 and float(dz[0, 0]) != 0.0
    with pytest.raises(ValueError):
        b200mdm.shape_sdf(0.0, 0.0)
    with pytest.raises(ValueError):
        b200mdm.shape_sdf(0.0, 0.0, boxes=[(1.0, 0.0, 0.0, 1.0)])
    with pytest.raises(ValueError):
        b200mdm.shape_sdf(0.0, 0.0, discs=[(0.0, 0.0, 0.0)])


def test_scene_grid_checks():
    g = b200mdm.SceneGrid(np.zeros((3, 4, 5)), (1, 2), 0.5)
    assert g.per_sample and g.shape == (4, 5) and g.origin == (1.0, 2.0) and g.cell == 0.5
    assert g.values.dtype == torch.float32
    assert torch.equal(g.shard(1, 3).values, g.values[1:3])
    shared = b200mdm.SceneGrid(torch.zeros(4, 5), (0, 0), 1)
    assert shared.shard(1, 2) is shared
    for bad in (dict(values=torch.zeros(4, 5, dtype=torch.int32)), dict(values=torch.zeros(5)),
                dict(values=torch.zeros(1, 2, 4, 5)), dict(values=torch.zeros(1, 5)), dict(values=torch.zeros(4, 1)),
                dict(values=torch.full((4, 5), float("nan"))), dict(values=torch.full((4, 5), 1e300, dtype=torch.float64)),
                dict(values=[[0.0, 1.0], [2.0, 3.0]]),
                dict(origin=(0.0, float("inf"))), dict(origin=(0.0, 0.0, 0.0)), dict(origin=(1e300, 0.0)),
                dict(cell=0.0), dict(cell=-1.0), dict(cell=float("nan")), dict(cell=float("inf")), dict(cell=1e-50)):
        kw = dict(dict(values=torch.zeros(4, 5), origin=(0.0, 0.0), cell=1.0), **bad)
        with pytest.raises(ValueError):
            b200mdm.SceneGrid(**kw)


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_wrapper_checks():
    model, diffusion = _model()
    mean, std = jo.motion_stats(263)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, floor_weight=FW, obstacle_weight=OW, obstacle_margin=R)
    assert jc.obstacle_weight == OW and jc.obstacle_margin == R
    for bad in (dict(obstacle_weight=-1.0), dict(obstacle_weight=float("nan")), dict(obstacle_margin=-0.1),
                dict(obstacle_margin=float("inf"))):
        with pytest.raises(ValueError):
            b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, **bad)
    B, T = 2, 24
    shape = (B, 263, 1, T)
    x = torch.zeros(shape)
    t = torch.zeros(B, dtype=torch.long)
    # with an obstacle weight the joint keys are optional
    obst = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, obstacle_weight=OW, obstacle_margin=R)
    c, w = obst.targets({}, shape)
    assert c.shape == (B, 22, 3, T) and float(w.abs().max()) == 0.0
    grid = b200mdm.SceneGrid(torch.zeros(4, 5), (0.0, 0.0), 0.5)
    y = {"text_embed": torch.zeros(1, B, 512), "scale": torch.ones(B), "obstacle_sdf": grid, "terrain": grid}
    snapshot = dict(y)
    assert jc.scene(y, shape) == (grid, grid)
    assert obst.scene({"obstacle_sdf": grid}, shape) == (grid, None)
    plain = b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 4, floor_weight=FW)
    assert plain.scene({"obstacle_sdf": grid}, shape) is None                 # no obstacle weight: the key is unread
    per = b200mdm.SceneGrid(torch.zeros(B + 1, 4, 5), (0.0, 0.0), 0.5)
    for wrapper, yy in ((obst, dict(y, obstacle_sdf=None)), (obst, {k: v for k, v in y.items() if k != "obstacle_sdf"}),
                        (obst, dict(y, terrain=None, obstacle_sdf=torch.zeros(4, 5))),
                        (jc, dict(y, terrain=torch.zeros(4, 5))), (jc, dict(y, obstacle_sdf=per)), (jc, dict(y, terrain=per)),
                        (obst, y)):                                         # a terrain with floor_weight 0
        for call in (lambda: diffusion.p_sample_loop(wrapper, shape, model_kwargs={"y": yy}),
                     lambda: diffusion.ddim_sample(wrapper, x, t, model_kwargs={"y": yy})):
            with pytest.raises(ValueError):
                call()
    assert y.keys() == snapshot.keys() and all(y[k] is snapshot[k] for k in y)
    # the refusals are joint control's
    with pytest.raises(NotImplementedError):
        diffusion.plms_sample_loop(jc, shape, model_kwargs={"y": y})
    with pytest.raises(NotImplementedError):
        diffusion.dpm_solver_sample_loop(jc, shape, model_kwargs={"y": y})
    with pytest.raises(TypeError):
        b200mdm.HandshakeSampleModel(jc, 4)


def test_shard_model_kwargs_slices_per_sample_grids():
    per = b200mdm.SceneGrid(torch.rand(6, 3, 4), (0.0, 1.0), 0.5)
    shared = b200mdm.SceneGrid(torch.rand(3, 4), (0.0, 1.0), 0.5)
    y = {"obstacle_sdf": per, "terrain": shared, "text_embed": torch.zeros(1, 6, 512)}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(part["obstacle_sdf"].values, per.values[2:5]) and part["obstacle_sdf"].origin == per.origin
    assert part["terrain"] is shared


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    f = ctypes.c_float
    buf = (ctypes.c_float * 64)()
    ok = _lib.Grid(ctypes.cast(buf, ctypes.c_void_p), 0, 4, 4, 0.0, 0.0, 0.5)
    assert lib.b200mdm_set_scene_guidance(None, f(1.0), f(0.2), ctypes.byref(ok), None, None) == _lib.EINVAL

    def grid(**kw):
        g = _lib.Grid(ctypes.cast(buf, ctypes.c_void_p), 0, 4, 4, 0.0, 0.0, 0.5)
        for k, v in kw.items():
            setattr(g, k, v)
        return g

    def hook(B=2, fw=1.0, ow=1.0, r=0.2, sdf=ok, terrain=None, step=1e-3):
        return lib.b200mdm_test_scene_guidance(buf, buf, buf, buf, buf, None, None, B, 60, 263, f(step), 4, f(0.0), f(fw),
                                               f(0.0), f(ow), f(r), None if sdf is None else ctypes.byref(sdf),
                                               None if terrain is None else ctypes.byref(terrain), buf, None, None)
    for kw, msg in ((dict(step=0.0), b"step"), (dict(ow=-1.0), b"obstacle weight"), (dict(ow=float("nan")), b"obstacle weight"),
                    (dict(r=-0.1), b"margin"), (dict(r=float("inf")), b"margin"), (dict(sdf=None), b"without an obstacle sdf"),
                    (dict(sdf=grid(values=None)), b"null values"), (dict(sdf=grid(gz=1)), b"cells"),
                    (dict(sdf=grid(gx=1)), b"cells"), (dict(terrain=grid(cell=0.0)), b"cell"),
                    (dict(terrain=grid(cell=float("nan"))), b"cell"), (dict(sdf=grid(x0=float("inf"))), b"origin"),
                    (dict(terrain=grid(z0=float("nan"))), b"origin"), (dict(sdf=grid(batch_stride=15)), b"batch stride"),
                    (dict(sdf=grid(batch_stride=-16)), b"batch stride"), (dict(B=3, sdf=grid(batch_stride=2 ** 62)), b"batch stride"),
                    (dict(fw=0.0, terrain=ok), b"floor weight")):
        assert hook(**kw) == _lib.EINVAL, kw
        assert msg in lib.b200mdm_last_error(), (kw, lib.b200mdm_last_error())


def test_symbols_in_header_and_lib():
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    assert "typedef struct b200mdm_grid" in header
    for name in ("b200mdm_set_scene_guidance", "b200mdm_test_scene_guidance"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)
