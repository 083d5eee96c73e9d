"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

fp64 restatement of the interaction terms of joint-position control (DESIGN.md, "Joint-position control", "Several
characters in one scene"): a batch of B motions is B / C scenes of C characters, motions [sC, sC + C) forming scene s.
Character a's motion p_a = recover_from_ric(x0_a * std + mean) (oracle/ric_oracle.py) stays in its own frame; its scene
placement (x, z, phi) = placement[a] maps it into the scene frame,

    Q_a = place_a(p_a):  (x, z) <- rot(phi) (x, z) + (X, Z),  y unchanged,
    rot(phi) (x, z) = (x cos phi - z sin phi, x sin phi + z cos phi),

the sense in which ric_rot(cos(phi / 2), sin(phi / 2), .) turns (ric_oracle._rot_y_inv; the root yaw's sense).  With
L_ab = min(L_a, L_b) and d = |Q_a[t, j] - Q_b[t, k]|, the energy adds

    G_inter = 1/2 la sum_scenes sum_{a<b} sum_{t<L_ab} sum_{j,k} max(r - d, 0)^2
            + 1/2 sum_n sum_{t<L_ab} w_n[t] max(|Q_{a_n}[t, j_n] - Q_{b_n}[t, k_n]| - delta_n, 0)^2

to the scene-guided G of oracle/scene_guidance_oracle.py.  Per sample, a pair's energy (an avoidance pair or a reach
row) belongs to its lower rank, as the kernel counts it.

`guide` takes the gradient with torch.autograd; `grad_manual` writes the interaction terms' position adjoint e out, from
each character's side as the kernel forms it (the avoidance gradient at d = 0 taken as 0), rotates it back by
rot(phi)^T and hands it to joint_control_oracle.grad_manual's chain, with the scene oracle's grad_manual for the other
terms and optional mutants for the tests' sensitivity checks.
"""
from typing import NamedTuple

import torch

from . import foot_guidance_oracle as fo
from . import joint_control_oracle as jo
from . import scene_guidance_oracle as so

# a partner read from the next scene; the placement rotation transposed; the margin's sign flipped; L_ab replaced by the
# character's own L_a; the reach gradient applied to the a side only; Gauss-Seidel reads (a partner's position taken
# after its own update in the same iteration: the missing cluster barrier)
MUTANTS = ("next_scene", "rot_transposed", "margin_sign", "length_a", "reach_one_side", "gauss_seidel")


class Inter(NamedTuple):
    """The interaction terms: C characters per scene, the avoidance weight and margin, placement [B, 3] (x, z, phi),
    pairs int [N, 4] scene-local (a, j, b, k), reach [N] and pair_weight [N, T] (every scene) or [B / C, N, T]."""
    C: int
    weight: float
    margin: float
    placement: torch.Tensor
    pairs: torch.Tensor = torch.zeros(0, 4, dtype=torch.int64)
    reach: torch.Tensor = torch.zeros(0, dtype=torch.float64)
    pair_weight: torch.Tensor = torch.zeros(0, 1, dtype=torch.float64)


class Scene(NamedTuple):
    """The terms of oracle/scene_guidance_oracle.py"""
    contact_w: float = 0.0
    floor_w: float = 0.0
    floor_h: float = 0.0
    obstacle_w: float = 0.0
    margin: float = 0.0
    sdf: object = None
    terrain: object = None


def place(p, placement, mutant=None):
    """Q [B, T, J, 3] of own-frame positions p [B, T, J, 3] (fp64)"""
    pl = placement.double()
    phi = -pl[:, 2] if mutant == "rot_transposed" else pl[:, 2]
    c, s = torch.cos(phi)[:, None, None], torch.sin(phi)[:, None, None]
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return torch.stack([c * x - s * z + pl[:, 0, None, None], y, s * x + c * z + pl[:, 1, None, None]], -1)


def _pair_weight(inter, S, T):
    w = inter.pair_weight.double()
    return (w if w.dim() == 3 else w.expand(S, -1, -1))[..., :T]                       # [S, N, T]


def _scene_lengths(lengths, B, T, C):
    return fo._lengths(lengths, B, T).reshape(B // C, C)                               # [S, C]


def inter_terms(p, inter, lengths=None):
    """G_inter per sample [B] (each pair's energy at its lower rank) of own-frame p [B, T, J, 3] (fp64,
    differentiable)."""
    B, T, J, _ = p.shape
    C, S = inter.C, B // inter.C
    Q = place(p, inter.placement).reshape(S, C, T, J, 3)
    L = _scene_lengths(lengths, B, T, C)
    t = torch.arange(T)
    G = torch.zeros(S, C, dtype=torch.float64)
    for a in range(C):
        for b in range(a + 1, C):
            live = (t[None, :] < torch.minimum(L[:, a], L[:, b])[:, None]).double()   # [S, T]
            if inter.weight > 0:
                d = (Q[:, a, :, :, None] - Q[:, b, :, None, :]).pow(2).sum(-1).sqrt()  # [S, T, J, J]
                m = torch.clamp(inter.margin - d, min=0.0)
                G[:, a] = G[:, a] + 0.5 * inter.weight * (live[:, :, None, None] * m * m).sum((1, 2, 3))
    pw = _pair_weight(inter, S, T)
    for n, (a, j, b, k) in enumerate(inter.pairs.tolist()):
        live = (t[None, :] < torch.minimum(L[:, a], L[:, b])[:, None]).double()
        d = (Q[:, a, :, j] - Q[:, b, :, k]).pow(2).sum(-1).sqrt()                       # [S, T]
        m = torch.clamp(d - float(inter.reach[n]), min=0.0)
        G[:, min(a, b)] = G[:, min(a, b)] + 0.5 * (pw[:, n] * live * m * m).sum(1)
    return G.reshape(B)


def loss(x0, mean, std, target, weight, scene, inter, kappa, lengths=None):
    """total G per sample [B] of x0 [B, D, T] (fp64, differentiable) with a fixed kappa [B, 4, T]"""
    G = so.loss(x0, mean, std, target, weight, *scene, kappa, lengths)
    return G + inter_terms(fo._positions(x0, mean, std), inter, lengths)


def guide(x0, mean, std, target, weight, step, iters, scene, inter, contact=None, lengths=None):
    """(guided x0 fp64 in x0's shape, total G fp64 [iters + 1, B]) by autograd; kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = fo._kappa(x0, mean, std, contact, lengths)
    losses = []
    for k in range(iters + 1):
        x.requires_grad_(True)
        G = loss(x, mean, std, target, weight, scene, inter, kappa, lengths)
        losses.append(G.detach())
        if k == iters:
            break
        (g,) = torch.autograd.grad(G.sum(), x)
        x = (x - step * g).detach()
    return x.detach().reshape(x0.shape), torch.stack(losses)


def inter_adjoint(p, inter, lengths=None, mutant=None):
    """(G_inter [B], its gradient in the own frames [B, T, J, 3]) of p [B, T, J, 3], from each character's side: the
    scene-frame gradient of every pair it belongs to, with the partners' positions as they are, rotated back by
    rot(phi)^T.  The avoidance gradient at d = 0 is 0."""
    B, T, J, _ = p.shape
    C, S = inter.C, B // inter.C
    Q = place(p, inter.placement, mutant).reshape(S, C, T, J, 3)
    Qp = torch.roll(Q, -1, 0) if mutant == "next_scene" else Q                          # the partners' positions
    L = _scene_lengths(lengths, B, T, C)
    r = -inter.margin if mutant == "margin_sign" else inter.margin
    t = torch.arange(T)

    def live(a, b):
        Lab = L[:, a] if mutant == "length_a" else torch.minimum(L[:, a], L[:, b])
        return (t[None, :] < Lab[:, None]).double()                                    # [S, T]

    G = torch.zeros(S, C, dtype=torch.float64)
    gQ = torch.zeros(S, C, T, J, 3, dtype=torch.float64)
    for a in range(C):
        for b in range(C):
            if a == b or inter.weight == 0:
                continue
            Dv = Q[:, a, :, :, None] - Qp[:, b, :, None, :]                               # [S, T, J, J, 3]
            d = Dv.pow(2).sum(-1).sqrt()
            m = torch.clamp(r - d, min=0.0) * live(a, b)[:, :, None, None]
            coef = torch.where(d > 0, inter.weight * m / torch.where(d > 0, d, torch.ones_like(d)), torch.zeros_like(d))
            gQ[:, a] -= (coef[..., None] * Dv).sum(3)
            if a < b:
                G[:, a] += 0.5 * inter.weight * (m * m).sum((1, 2, 3))
    pw = _pair_weight(inter, S, T)
    for n, (a, j, b, k) in enumerate(inter.pairs.tolist()):
        for me, mj, other, ok in ((a, j, b, k), (b, k, a, j)):
            if mutant == "reach_one_side" and me == b:
                continue
            Dv = Q[:, me, :, mj] - Qp[:, other, :, ok]                                      # [S, T, 3]
            d = Dv.pow(2).sum(-1).sqrt()
            m = torch.clamp(d - float(inter.reach[n]), min=0.0) * live(me, other)
            gQ[:, me, :, mj] += (pw[:, n] * m / torch.where(d > 0, d, torch.ones_like(d)))[..., None] * Dv
            if me == min(a, b):
                G[:, me] += 0.5 * (pw[:, n] * m * m).sum(1)
    gQ = gQ.reshape(B, T, J, 3)
    pl = inter.placement.double()
    phi = -pl[:, 2] if mutant == "rot_transposed" else pl[:, 2]
    c, s = torch.cos(phi)[:, None, None], torch.sin(phi)[:, None, None]
    e = torch.stack([c * gQ[..., 0] + s * gQ[..., 2], gQ[..., 1], -s * gQ[..., 0] + c * gQ[..., 2]], -1)
    return G.reshape(B), e


def grad_manual(x0, mean, std, target, weight, scene, inter, contact=None, lengths=None, mutant=None, kappa=None):
    """(G [B], dG/dx0 [B, D, T]) in fp64: the interaction terms' position adjoint e (inter_adjoint) through
    joint_control_oracle.grad_manual's chain, plus scene_guidance_oracle.grad_manual for the other terms.
    mutant: None or one of MUTANTS but 'gauss_seidel' (guide_manual's)."""
    x0 = jo._flat(x0)
    B, D, T = x0.shape
    J = jo.n_joints(D)
    if kappa is None:
        kappa = fo._kappa(x0, mean, std, contact, lengths)
    G, g = so.grad_manual(x0, mean, std, target, weight, *scene, contact, lengths, None, kappa)
    p = fo._positions(x0, mean, std)                                                     # [B, T, J, 3]
    Gi, e = inter_adjoint(p, inter, lengths, mutant)
    _, gi = jo.grad_manual(x0, mean, std, (p - e).permute(0, 2, 3, 1), torch.ones(B, J, T, dtype=torch.float64))
    return G + Gi, g + gi


def guide_manual(x0, mean, std, target, weight, step, iters, scene, inter, contact=None, lengths=None, mutant=None):
    """guide() through grad_manual; mutant as there, or 'gauss_seidel': within an iteration rank 0's characters step
    first, then rank 1's from the updated rank 0, and so on.  kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = fo._kappa(x0, mean, std, contact, lengths)
    rank = torch.arange(x.shape[0]) % inter.C
    losses = []
    for k in range(iters + 1):
        G, g = grad_manual(x, mean, std, target, weight, scene, inter, contact, lengths,
                           None if mutant == "gauss_seidel" else mutant, kappa)
        losses.append(G)
        if k == iters:
            break
        if mutant != "gauss_seidel":
            x = x - step * g
            continue
        for c in range(inter.C):
            if c > 0:
                _, g = grad_manual(x, mean, std, target, weight, scene, inter, contact, lengths, None, kappa)
            x = torch.where((rank == c)[:, None, None], x - step * g, x)
    return x.reshape(x0.shape), torch.stack(losses)


def guided_denoiser(denoise, mean, std, target, weight, step, iters, scene, inter, contact=None, lengths=None):
    """denoise(x, i) followed by the guidance of its x0 (fp64, rounded back to x0's dtype)."""
    def f(x, i):
        x0 = denoise(x, i)
        with torch.enable_grad():
            g, _ = guide(x0, mean, std, target, weight, step, iters, scene, inter, contact, lengths)
        return g.to(x0.dtype)
    return f


def step_bound(std, weight, extent, T, scene, inter, kappa_max=1.0):
    """The step size the tests use, 1 / L_GN with the interaction terms (DESIGN.md, "Several characters in one scene"):
    the scene bound's L_GN (scene_guidance_oracle.step_bound) plus s^2 (4 la J^2 (C - 1) + 4 N w_max) T g, with
    g = 1 + T (1 + 4 A^2) and w_max the largest pair weight.  Each distance has a unit gradient in the scene frame, the
    placement is a rotation, and a pair couples two characters (the factor 2 of |u u^T| over both sides, times the 2 of
    the obstacle term's bound); avoidance can act on all J^2 joint pairs against C - 1 partners at every frame."""
    J = jo.n_joints(std.shape[0])
    R = jo.ric_features(J)
    s2 = float(std[:R].double().max()) ** 2
    W = float(weight.double().sum((1, 2)).max())
    gain = 1 + T * (1 + 4 * extent ** 2)
    lf = scene.floor_w if scene.terrain is None else 2 * scene.floor_w * (1 + 2 * so.max_slope(scene.terrain) ** 2 * J * T * gain)
    lo = 0.0 if scene.sdf is None else 2 * scene.obstacle_w * so.max_slope(scene.sdf) ** 2 * J * T * gain
    wmax = float(inter.pair_weight.double().max()) if inter.pair_weight.numel() else 0.0
    N = int(inter.pairs.shape[0])
    li = (4 * inter.weight * J * J * (inter.C - 1) + 4 * N * wmax) * T * gain
    return 1.0 / (s2 * (W * gain + 4 * scene.contact_w * kappa_max * (3 + 4 * extent ** 2) + lf + lo + li))
