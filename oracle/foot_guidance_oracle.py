"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

fp64 restatement of the foot-contact and floor terms of joint-position control (DESIGN.md, "Joint-position control",
"Foot contact and floor"):

    G = G_joint + 1/2 lc sum_{k<4, t<T-1} kappa_k[t] |p[t+1, f_k] - p[t, f_k]|^2
                + 1/2 lf sum_{t<L, j} min(p[t, j].y - h, 0)^2,

p = recover_from_ric(x0 * std + mean) (oracle/ric_oracle.py), G_joint as oracle/joint_control_oracle.py states it.
kappa is y['foot_contact'] or, derived, 1 where the de-normalised contact feature k of frame t is > 0.5 and t + 1 < L.

`guide` takes the gradient with torch.autograd; `grad_manual` writes the foot terms' position adjoint out as the kernel
forms it (csrc/joint_guidance.cuh) and hands it to joint_control_oracle.grad_manual's chain, with optional mutants for the
tests' sensitivity checks.  `guided_denoiser` wraps a denoise(x, i) of the oracles as joint_control_oracle's does.
"""
import torch

from . import joint_control_oracle as jo
from . import ric_oracle

FOOT_JOINTS = {22: (7, 10, 8, 11), 21: (19, 20, 14, 15)}   # contact channels D - 4 .. D - 1 (feet_l, then feet_r)
MUTANTS = ("kappa_shift", "swap", "delta_sign", "floor_max", "no_lengths")


def _lengths(lengths, B, T):
    if lengths is None:
        return torch.full((B,), T, dtype=torch.int64)
    return torch.as_tensor(lengths).reshape(-1).to(torch.int64).clamp(0, T)


def derive_contact(x0, mean, std, lengths=None):
    """kappa [B, 4, T] fp64 of normalised x0 [B, D, T]: 1 where the de-normalised contact feature is > 0.5 at frame t
    and t + 1 < L_b, else 0 (the last frame has no pair).  The de-normalisation is rounded as the kernel's (fp32)."""
    x0 = jo._flat(x0)
    B, D, T = x0.shape
    x = (x0[:, D - 4:].float() * std[D - 4:].float()[None, :, None] + mean[D - 4:].float()[None, :, None])
    t = torch.arange(T)
    live = (t[None, :] + 1 < _lengths(lengths, B, T)[:, None])
    return ((x > 0.5) & live[:, None, :]).double()


def _kappa(x0, mean, std, contact, lengths, mutant=None):
    B, D, T = jo._flat(x0).shape
    if contact is None:
        k = derive_contact(x0, mean, std, None if mutant == "no_lengths" else lengths)
    else:
        k = contact.double().clone()
    k[:, :, T - 1:] = 0                                          # pair (t, t + 1) needs frame t + 1
    if mutant == "kappa_shift":                                  # channel t applied to the pair (t - 1, t)
        k = torch.cat([k[:, :, 1:], torch.zeros_like(k[:, :, :1])], -1)
    if mutant == "swap":                                         # left and right channels swapped
        k = k[:, [2, 3, 0, 1]]
    return k


def _positions(x0, mean, std):
    """p [B, T, J, 3] fp64 of normalised x0 [B, D, T] (differentiable)"""
    D = x0.shape[1]
    data = (x0 * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    return ric_oracle.recover_from_ric(data, jo.n_joints(D))


def foot_terms(x0, mean, std, kappa, contact_w, floor_w, floor_h, lengths=None):
    """(contact energy [B], floor energy [B]) of normalised x0 [B, D, T] (fp64, differentiable) with kappa [B, 4, T]."""
    B, D, T = x0.shape
    p = _positions(x0, mean, std)
    f = list(FOOT_JOINTS[jo.n_joints(D)])
    d = p[:, 1:, f] - p[:, :-1, f]                                                   # [B, T-1, 4, 3]
    ec = 0.5 * contact_w * (kappa[:, :, :T - 1].permute(0, 2, 1) * (d * d).sum(-1)).sum((1, 2))
    live = (torch.arange(T)[None, :] < _lengths(lengths, B, T)[:, None]).double()    # [B, T]
    m = torch.clamp(p[..., 1] - floor_h, max=0.0)                                    # [B, T, J]
    ef = 0.5 * floor_w * (live[:, :, None] * m * m).sum((1, 2))
    return ec, ef


def loss(x0, mean, std, target, weight, contact_w, floor_w, floor_h, kappa, lengths=None):
    """total G per sample [B] of x0 [B, D, T] (fp64, differentiable) with a fixed kappa [B, 4, T]"""
    ec, ef = foot_terms(x0, mean, std, kappa, contact_w, floor_w, floor_h, lengths)
    return jo.loss(x0, mean, std, target, weight) + ec + ef


def guide(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h=0.0, contact=None, lengths=None):
    """(guided x0 fp64 in x0's shape, total G fp64 [iters + 1, B]) by autograd; kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = _kappa(x0, mean, std, contact, lengths)
    losses = []
    for k in range(iters + 1):
        x.requires_grad_(True)
        G = loss(x, mean, std, target, weight, contact_w, floor_w, floor_h, kappa, lengths)
        losses.append(G.detach())
        if k == iters:
            break
        (g,) = torch.autograd.grad(G.sum(), x)
        x = (x - step * g).detach()
    return x.detach().reshape(x0.shape), torch.stack(losses)


def grad_manual(x0, mean, std, target, weight, contact_w, floor_w, floor_h=0.0, contact=None, lengths=None, mutant=None,
                kappa=None):
    """(G [B], dG/dx0 [B, D, T]) in fp64: the position adjoint e of DESIGN.md, the joint term's plus
    lc (kappa[t-1] Delta[t-1] - kappa[t] Delta[t]) at (t, f_k) and lf min(p.y - h, 0) in y, through
    joint_control_oracle.grad_manual's chain (unit weights on every joint and the target p - e have position adjoint e).
    mutant: None or one of MUTANTS (kappa on the pair (t-1, t), left / right swapped, Delta's sign flipped in the
    adjoint, max for min in the floor term, lengths ignored)."""
    x0 = jo._flat(x0)
    B, D, T = x0.shape
    J = jo.n_joints(D)
    if kappa is None:
        kappa = _kappa(x0, mean, std, contact, lengths, mutant)
    p = _positions(x0, mean, std).permute(0, 2, 3, 1)                              # [B, J, 3, T]
    c_t, w = target.double(), weight.double()
    d = torch.where(w[:, :, None] != 0, p - c_t, torch.zeros_like(p))
    e = w[:, :, None] * d
    Lb = _lengths(None if mutant == "no_lengths" else lengths, B, T)
    live = (torch.arange(T)[None, :] < Lb[:, None]).double()                       # [B, T]
    m = torch.clamp(p[:, :, 1] - floor_h, min=0.0) if mutant == "floor_max" else torch.clamp(p[:, :, 1] - floor_h, max=0.0)
    e[:, :, 1] += floor_w * live[:, None] * m
    f = list(FOOT_JOINTS[J])
    delta = p[:, f, :, 1:] - p[:, f, :, :-1]                                         # [B, 4, 3, T-1]
    kd = kappa[:, :, None, :T - 1] * delta
    ce = torch.zeros(B, 4, 3, T, dtype=torch.float64)
    ce[..., 1:] += kd
    ce[..., :-1] -= kd
    e[:, f] += -contact_w * ce if mutant == "delta_sign" else contact_w * ce
    G = 0.5 * (w[:, :, None] * d * d).sum((1, 2, 3)) + 0.5 * contact_w * (kd * delta).sum((1, 2, 3)) + \
        0.5 * floor_w * (live[:, None] * m * m).sum((1, 2))
    _, g = jo.grad_manual(x0, mean, std, p - e, torch.ones(B, J, T, dtype=torch.float64))
    return G, g


def guide_manual(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h=0.0, contact=None, lengths=None,
                 mutant=None):
    """guide() through grad_manual; mutant as there.  kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = _kappa(x0, mean, std, contact, lengths, mutant)
    losses = []
    for k in range(iters + 1):
        G, g = grad_manual(x, mean, std, target, weight, contact_w, floor_w, floor_h, contact, lengths, mutant, kappa)
        losses.append(G)
        if k == iters:
            break
        x = x - step * g
    return x.reshape(x0.shape), torch.stack(losses)


def guided_denoiser(denoise, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h=0.0, contact=None,
                    lengths=None):
    """denoise(x, i) followed by the guidance of its x0 (fp64, rounded back to x0's dtype)."""
    def f(x, i):
        x0 = denoise(x, i)
        with torch.enable_grad():
            g, _ = guide(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h, contact, lengths)
        return g.to(x0.dtype)
    return f


def step_bound(std, weight, extent, T, contact_w, floor_w, kappa_max=1.0):
    """The step size the tests use, 1 / L_GN with the foot terms (DESIGN.md, "Foot contact and floor"):
    L_GN = s^2 (W (1 + T (1 + 4 A^2)) + 4 lc kappa_max (3 + 4 A^2) + lf), with s, W and A as in
    joint_control_oracle.step_bound and kappa_max the largest contact weight (1 for a derived mask)."""
    R = jo.ric_features(jo.n_joints(std.shape[0]))
    s2 = float(std[:R].double().max()) ** 2
    W = float(weight.double().sum((1, 2)).max())
    return 1.0 / (s2 * (W * (1 + T * (1 + 4 * extent ** 2)) + 4 * contact_w * kappa_max * (3 + 4 * extent ** 2) + floor_w))
