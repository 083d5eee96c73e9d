"""CPU: goal-directed autoregressive chains (DESIGN.md, "Goals in the world frame").

  * the fp64 oracle (oracle/goal_oracle.py) maps every W-frame target of the reference fixture onto the chunk-local
    target the reference computes from the chunk alone (tests/golden/goal_frames.npz);
  * AutoRegressiveSampler's ValueErrors for keys that clash, before any engine work and with y unmodified;
  * the new C symbols, and their argument checks without a device."""
import ctypes
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import default_args
from oracle import goal_oracle as go

EXT = ["pelvis", "left_foot", "right_foot", "left_wrist", "right_wrist", "head", "traj", "heading"]


def _case(golden, case):
    z = golden("goal_frames.npz")
    off = int(z["ctx"]) if case == "prefix" else 0
    return z, off, int(z["pred"]), int(z["n_chunks"])


@pytest.mark.parametrize("case", ["prefix", "noprefix"])
def test_oracle_maps_world_onto_chunk_local(golden, case):
    z, off, pred, n = _case(golden, case)
    mean, std, motion = (torch.from_numpy(z[k]) for k in ("mean", "std", case + "_motion"))
    names = [[j for j in str(s).split(";") if j] for s in z["names"]]
    checked = 0
    for c in range(n):
        fr = go.frame_at(motion, mean, std, off + c * pred)
        world = torch.from_numpy(z["%s_world_%d" % (case, c)])
        local = torch.from_numpy(z["%s_local_%d" % (case, c)]).double()
        got = go.to_chunk(world, fr)
        back = go.to_world(got, fr)
        for b in range(world.shape[0]):
            for j in names[b]:
                i = EXT.index(j)
                assert float((got[b, i] - local[b, i]).norm() / local[b, i].norm()) < 1e-5, (c, b, j)
                assert float((back[b, i] - world[b, i].double()).norm()) < 1e-12
                checked += 1
            if z["is_heading"][b]:
                d = float(got[b, -1, 0] - local[b, -1, 0])
                assert abs((d + math.pi) % (2 * math.pi) - math.pi) < 1e-5, (c, b)
                assert -math.pi < float(got[b, -1, 0]) <= math.pi
                checked += 1
        if c == 0 and off == 0:                      # M_0 is the identity
            assert torch.equal(got[:, :-1], world[:, :-1].double())
    assert checked >= 30


def test_oracle_frame_is_nontrivial(golden):
    z, off, pred, n = _case(golden, "prefix")
    mean, std, motion = (torch.from_numpy(z[k]) for k in ("mean", "std", "prefix_motion"))
    fr = go.frame_at(motion, mean, std, off + (n - 1) * pred)
    assert float(fr["yaw"].abs().min()) > 0.1 and float(fr["P"].norm(dim=1).min()) > 0.1
    carry = go.carry_after(motion, mean, std, off)
    assert torch.allclose(go.frame_at(motion, mean, std, off)["yaw"], carry[:, 0], rtol=0, atol=1e-12)


def _dip(target=True, encoder="multi"):
    over = dict(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert", context_len=4, pred_len=8)
    if target:
        over.update(multi_target_cond=True, multi_encoder_type=encoder, target_enc_layers=1)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    return model, diffusion


def _y(B=2, n_ext=8):
    tg = b200mdm.synthetic_target_inputs(B, seed=5)
    return dict(prefix=torch.zeros(B, 263, 1, 4), text_embed=(torch.zeros(3, B, 768), torch.zeros(B, 3, dtype=torch.bool)),
                lengths=torch.full((B,), 8), mask=torch.ones(B, 1, 1, 8, dtype=torch.bool),
                target_world=torch.zeros(B, n_ext, 3), target_joint_names=tg["target_joint_names"],
                is_heading=tg["is_heading"])


@pytest.mark.parametrize("what", ["with_target_cond", "no_encoder", "no_mean_std", "chunk_axis", "bad_shape",
                                  "bad_joint", "bad_mean"])
def test_sampler_value_errors(what):
    model, diffusion = _dip(target=what != "no_encoder")
    y = _y()
    mean, std = torch.zeros(263), torch.ones(263)
    if what == "with_target_cond":
        y["target_cond"] = torch.zeros(2, 8, 3)
    if what == "no_mean_std":
        mean = std = None
    if what == "chunk_axis":                         # required 24 / pred 8: 3 chunks
        y["target_world"] = torch.zeros(2, 2, 8, 3)
    if what == "bad_shape":
        y["target_world"] = torch.zeros(2, 7, 3)
    if what == "bad_joint":
        y["target_joint_names"] = [["elbow"], []]
    if what == "bad_mean":
        mean = torch.zeros(251)
    before = dict(y)
    calls = []

    def sample_fn(*a, **k):                          # never reached: the checks come first
        calls.append(1)
        raise AssertionError("sampled")
    args = SimpleNamespace(pred_len=8, context_len=4, autoregressive_include_prefix=False)
    s = b200mdm.AutoRegressiveSampler(args, sample_fn, 24, mean=mean, std=std)
    with pytest.raises(ValueError):
        s.sample(model, (2, 263, 1, 8), model_kwargs={"y": y})
    assert not calls
    assert y.keys() == before.keys() and all(y[k] is before[k] for k in y)


def test_shard_model_kwargs_slices_goals():
    for g in (torch.arange(4 * 8 * 3.0).view(4, 8, 3), torch.arange(3 * 4 * 8 * 3.0).view(3, 4, 8, 3)):
        out = parallel.shard_model_kwargs({"y": {"target_world": g}}, 1, 3)["y"]["target_world"]
        assert torch.equal(out, g[1:3] if g.dim() == 3 else g[:, 1:3])


def test_symbols_in_header_and_lib():
    import os
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "b200mdm.h")).read()
    for name in ("b200mdm_chain_set_goal", "b200mdm_chunk_frame"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_double * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    valid = (ctypes.c_uint8 * 64)()
    assert lib.b200mdm_chain_set_goal(None, p, p, p, 1, valid, None) == _lib.EINVAL
    good = dict(carry=p, frames=p, B=2, D=263, n=8, mean=p, std=p, goal=p, n_ext=8, out=p)

    def call(**over):
        a = dict(good, **over)
        return lib.b200mdm_chunk_frame(a["carry"], a["frames"], a["B"], a["D"], a["n"], a["mean"], a["std"], a["goal"],
                                       a["n_ext"], a["out"], None)
    for over in (dict(carry=None), dict(frames=None), dict(mean=None), dict(std=None), dict(goal=None), dict(out=None),
                 dict(B=0), dict(D=3), dict(n=-1), dict(n=257), dict(n_ext=1), dict(n_ext=65)):
        assert call(**over) == _lib.EINVAL, over
