"""Test inputs of the interaction terms of joint-position control, shared by tests/test_interaction_guidance_cpu.py and
tests/test_interaction_guidance_gpu.py: two scenes of C characters standing close together (so that avoidance acts
on many joint pairs), with reach rows between wrists, knees and feet and lengths that differ per character."""
import math

import torch

from oracle import foot_guidance_oracle as fo
from oracle import interaction_guidance_oracle as io
from oracle import joint_control_oracle as jo
from oracle import ric_oracle

LA, RA = 4.0, 0.3           # the avoidance weight and margin
EPS_G = 2.0 ** -12
U32 = 2.0 ** -24


def rows(D, C):
    """reach rows (a, j, b, k) valid for HumanML3D and KIT: a hand to a hand, a knee to a foot, across the scene"""
    r = [(0, 15, 1, 20), (1, 4, 0, 10), (C - 1, 18, 0, 19)]
    return torch.tensor(r if C > 2 else r[:2], dtype=torch.int64)


def case(D, T, C, seed, S=2, spacing=0.12, per_scene=True):
    """(x0 fp32 [S C, D, T], mean, std, Inter, lengths): the characters of a scene on a circle of chord `spacing`,
    each turned by its own phi"""
    g = torch.Generator().manual_seed(seed)
    B = S * C
    mean, std = jo.motion_stats(D)
    x0 = (torch.randn(B, D, T, generator=g) * 0.3).float()
    ang = 2 * math.pi * torch.arange(C, dtype=torch.float64) / C
    rad = spacing / (2 * math.sin(math.pi / C))
    pl = torch.stack([rad * torch.cos(ang), rad * torch.sin(ang), ang + 0.4], 1).repeat(S, 1)
    pl[:, :2] += 0.05 * torch.randn(B, 2, generator=g, dtype=torch.float64)
    pl = pl.float().double()
    pr = rows(D, C)
    N = pr.shape[0]
    reach = torch.tensor([0.05, 0.1, 0.0][:N], dtype=torch.float64)
    pw = torch.rand(S, N, T, generator=g, dtype=torch.float64) * 3.0
    pw[:, :, ::5] = 0.0
    pw = pw.float().double()
    if not per_scene:
        pw = pw[0]
    lengths = torch.tensor([T - (b % 3) * 5 for b in range(B)])
    return x0, mean, std, io.Inter(C, LA, RA, pl, pr, reach, pw), lengths


def extent(x0, mean, std, inter):
    p = fo._positions(x0.double(), mean, std)
    Q = io.place(p, inter.placement)
    return float(Q[..., [0, 2]].max() - Q[..., [0, 2]].min()) + 1.0


def kink_distance(x0, mean, std, inter, lengths):
    """the least distance (m) of a live pair from its kinks: |d - r| and d for avoidance, |d - delta| for reach rows"""
    B, D, T = x0.shape
    p = fo._positions(x0.double(), mean, std)
    C, S = inter.C, B // inter.C
    Q = io.place(p, inter.placement).reshape(S, C, T, -1, 3)
    L = fo._lengths(lengths, B, T).reshape(S, C)
    t = torch.arange(T)
    best = math.inf
    for a in range(C):
        for b in range(a + 1, C):
            live = t[None, :] < torch.minimum(L[:, a], L[:, b])[:, None]
            d = (Q[:, a, :, :, None] - Q[:, b, :, None, :]).pow(2).sum(-1).sqrt()[live]
            if d.numel():
                best = min(best, float((d - inter.margin).abs().min()), float(d.min()))
    for n, (a, j, b, k) in enumerate(inter.pairs.tolist()):
        live = t[None, :] < torch.minimum(L[:, a], L[:, b])[:, None]
        d = (Q[:, a, :, j] - Q[:, b, :, k]).pow(2).sum(-1).sqrt()[live]
        if d.numel():
            best = min(best, float((d - float(inter.reach[n])).abs().min()))
    return best


def step(x0, mean, std, inter, scene=io.Scene()):
    T, J = x0.shape[-1], jo.n_joints(x0.shape[1])
    return io.step_bound(std, torch.zeros(1, J, T), extent(x0, mean, std, inter), T, scene, inter)


def bound(want, x0, K):
    """the joint-control bound of DESIGN.md: 2^-12 max|x0_o - x0| + 2 u K max|x0|"""
    return EPS_G * float((want - x0.double()).abs().max()) + 2 * U32 * K * float(x0.abs().max())


def positions(x0, mean, std):
    return ric_oracle.recover_from_ric((x0.double() * std.double()[None, :, None] + mean.double()[None, :, None])
                                       .permute(0, 2, 1), jo.n_joints(x0.shape[1]))
