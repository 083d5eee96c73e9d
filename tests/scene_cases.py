"""Test inputs of the scene terms of joint-position control, shared by tests/test_scene_guidance_cpu.py and
tests/test_scene_guidance_gpu.py: motions with curved grids placed clear of their grid lines, and motions with
per-sample planar grids (whose bilinear gradient is continuous, so fp32 and fp64 pick equivalent cells)."""
import math

import torch

import b200mdm
from oracle import foot_guidance_oracle as fo
from oracle import joint_control_oracle as jo
from oracle import scene_guidance_oracle as so

CW, FW, FH, OW, R = 3.0, 5.0, -0.2, 2.0, 0.3


def _planar(B, gz, gx, origin, cell, slopes):
    """[B, gz, gx] grids a + sx x + sz z, one (a, sx, sz) per sample: bilinear sampling is exact and its gradient
    continuous across grid lines"""
    z = origin[1] + cell * torch.arange(gz, dtype=torch.float64)
    x = origin[0] + cell * torch.arange(gx, dtype=torch.float64)
    return torch.stack([a + sx * x[None, :] + sz * z[:, None] for a, sx, sz in slopes[:B]])


def _curved(p, shift):
    """an obstacle SDF (discs and a box near the motion) and a bumpy terrain, origin shifted by `shift` cells"""
    cell = 0.2
    o = (float(p[..., 0].min()) - 1.0 + shift * cell, float(p[..., 2].min()) - 1.0 + shift * cell)
    gz, gx = int((float(p[..., 2].max()) - o[1]) / cell) + 4, int((float(p[..., 0].max()) - o[0]) / cell) + 4
    cx, cz = float(p[..., 0].mean()), float(p[..., 2].mean())
    sdf = b200mdm.SceneGrid.from_shapes((gz, gx), o, cell, discs=[(cx, cz, 0.1), (cx + 0.5, cz - 0.3, 0.05)],
                                        boxes=[(cx - 0.6, cz + 0.2, cx - 0.5, cz + 0.4)])
    zz = o[1] + cell * torch.arange(gz, dtype=torch.float64)[:, None]
    xx = o[0] + cell * torch.arange(gx, dtype=torch.float64)[None, :]
    terrain = b200mdm.SceneGrid(0.15 * torch.sin(3 * xx) * torch.cos(2 * zz) + 0.05 * xx - 0.25, o, cell)
    return sdf, terrain


def line_distance(grid, p, active):
    """the least distance, in cells, from a grid line of the joints `active` marks (p [B, T, J, 3]), inside the grid"""
    u = (p[..., 0] - grid.origin[0]) / grid.cell
    v = (p[..., 2] - grid.origin[1]) / grid.cell
    d = torch.minimum((u - u.round()).abs(), (v - v.round()).abs())
    return float(d[active].min()) if bool(active.any()) else math.inf


def _active(x0, mean, std, sdf, terrain, lengths):
    """joints [B, T, J] the obstacle or terrain term acts on"""
    B, D, T = x0.shape
    p = fo._positions(x0, mean, std)
    live = (torch.arange(T)[None, :] < fo._lengths(lengths, B, T)[:, None])[..., None]
    flat = p.reshape(B, -1, 3)
    S = so.sample(sdf, flat[..., 0], flat[..., 2])[0].reshape(p.shape[:3])
    H = so.sample(terrain, flat[..., 0], flat[..., 2])[0].reshape(p.shape[:3])
    return p, live & (R - S > 0), live & (p[..., 1] - FH - H < 0)


def curved_case(D, T, seed, B=2):
    """x0 and curved grids such that the active joints keep >= 1e-3 cell from every grid line (the origin is moved by a
    fraction of a cell until they do)"""
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    x0 = torch.randn(B, D, T, generator=g, dtype=torch.float64) * 0.7
    target = torch.randn(B, J, 3, T, generator=g, dtype=torch.float64)
    weight = (torch.rand(B, J, T, generator=g) < 0.3).double()
    lengths = torch.tensor([T, max(1, T - 7)])[:B]
    p0 = fo._positions(x0, mean, std)
    for n in range(256):
        sdf, terrain = _curved(p0, (n * 0.618034) % 1.0)
        p, ao, af = _active(x0, mean, std, sdf, terrain, lengths)
        if min(line_distance(sdf, p, ao), line_distance(terrain, p, af)) >= 1e-3:
            return x0, mean, std, target, weight, lengths, sdf, terrain, int(ao.sum()), int(af.sum())
    raise AssertionError("no grid placement keeps the active joints 1e-3 cell from the grid lines")


def planar_case(D, T, seed, B=2):
    """x0 and per-sample planar grids with different x and z slopes, part of the motion outside them"""
    g = torch.Generator().manual_seed(seed)
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    x0 = torch.randn(B, D, T, generator=g, dtype=torch.float64) * 0.7
    target = torch.randn(B, J, 3, T, generator=g, dtype=torch.float64)
    o, c = (-2.0, -1.5), 0.25
    sdf = b200mdm.SceneGrid(_planar(B, 12, 14, o, c, [(0.3, 0.8, -0.5), (0.1, -0.6, 0.7), (0.2, 0.5, 0.5)]), o, c)
    terrain = b200mdm.SceneGrid(_planar(B, 12, 14, o, c, [(0.05, 0.3, 0.2), (-0.1, -0.2, 0.4), (0.0, 0.25, -0.3)]), o, c)
    lengths = torch.tensor([T, max(1, T - 7), max(1, T // 2)])[:B]
    return x0, mean, std, target, torch.zeros(B, J, T, dtype=torch.float64), lengths, sdf, terrain
