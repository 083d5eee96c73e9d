"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

fp64 restatement of joint-position control (DESIGN.md, "Joint-position control"; no reference counterpart):

    x = x0 * std + mean,   p = recover_from_ric(x, J)  (oracle/ric_oracle.py),
    G(x0) = 1/2 sum_{t,j} w[j,t] |p[t,j] - c[j,:,t]|^2,   K steps  x0 <- x0 - step * grad G(x0).

`guide` takes the gradient with torch.autograd through ric_oracle; `guide_manual` writes the forward and adjoint scans
out as the kernel runs them (csrc/joint_guidance.cuh), with optional mutants for the tests' sensitivity checks.
`guided_denoiser` wraps any denoise(x, i) of the oracles (plms_oracle.enc_denoiser, dec_emb_oracle.denoiser) so that
dec_emb_oracle.sample_loop gives the guided DDPM / DDIM loop: guidance acts on the model's x0, ahead of inpainting.
"""
import torch

from . import ric_oracle


def n_joints(D):
    return 22 if D == 263 else 21


def ric_features(J):
    """R: the features recover_from_ric reads (yaw velocity, XZ velocity, height, root-relative joints)."""
    return 4 + 3 * (J - 1)


def _flat(x0):
    """[B, D, T] or [B, D, 1, T] -> fp64 [B, D, T]"""
    return x0.reshape(x0.shape[0], x0.shape[1], x0.shape[-1]).double()


def loss(x0, mean, std, target, weight):
    """G per sample [B] of x0 [B, D, T] (fp64, differentiable)."""
    D = x0.shape[1]
    data = (x0 * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)   # [B, T, D]
    p = ric_oracle.recover_from_ric(data, n_joints(D))                                            # [B, T, J, 3]
    c = target.double().permute(0, 3, 1, 2)                                                       # [B, T, J, 3]
    w = weight.double().permute(0, 2, 1)                                                          # [B, T, J]
    d = torch.where(w[..., None] != 0, p - c, torch.zeros_like(p))                               # free joints: c unread
    return 0.5 * (w * (d * d).sum(-1)).sum((1, 2))


def guide(x0, mean, std, target, weight, step, iters):
    """(guided x0 fp64 in x0's shape, losses fp64 [iters + 1, B]) by autograd."""
    x = _flat(x0).clone()
    losses = []
    for k in range(iters + 1):
        x.requires_grad_(True)
        G = loss(x, mean, std, target, weight)
        losses.append(G.detach())
        if k == iters:
            break
        (g,) = torch.autograd.grad(G.sum(), x)
        x = (x - step * g).detach()
    return x.detach().reshape(x0.shape), torch.stack(losses)


def _rot(c, s, ax, az):
    """qrot(qinv((c, 0, s, 0)), (ax, *, az)) in x / z (ric_oracle._rot_y_inv)"""
    return ax + 2 * (c * (-s * az) - s * s * ax), az + 2 * (c * (s * ax) - s * s * az)


def grad_manual(x0, mean, std, target, weight, mutant=None):
    """(G [B], dG/dx0 [B, D, T]) in fp64 by the kernel's forward and adjoint scans.  mutant: None, 'no_yaw' (the yaw
    adjoint dropped), 'vel_shift' (the root-velocity adjoint handed to frame t instead of t - 1) or 'no_std' (std left
    out of the chain rule)."""
    x0 = _flat(x0)
    B, D, T = x0.shape
    J = n_joints(D)
    R = ric_features(J)
    sd = std.double()[None, :, None]
    x = x0 * sd + mean.double()[None, :, None]
    c_t = target.double()                                    # [B, J, 3, T]
    w = weight.double()                                      # [B, J, T]
    yaw = torch.zeros(B, T, dtype=torch.float64)
    yaw[:, 1:] = torch.cumsum(x[:, 0, :-1], -1)
    c, s = torch.cos(yaw), torch.sin(yaw)
    wx, wz = torch.zeros(B, T, dtype=torch.float64), torch.zeros(B, T, dtype=torch.float64)
    wx[:, 1:], wz[:, 1:] = _rot(c[:, 1:], s[:, 1:], x[:, 1, :-1], x[:, 2, :-1])
    px, pz = torch.cumsum(wx, -1), torch.cumsum(wz, -1)
    q = x[:, 4:R].reshape(B, J - 1, 3, T)
    rx, rz = _rot(c[:, None], s[:, None], q[:, :, 0], q[:, :, 2])
    p = torch.stack([torch.cat([px[:, None], rx + px[:, None]], 1), torch.cat([x[:, 3:4], q[:, :, 1]], 1),
                     torch.cat([pz[:, None], rz + pz[:, None]], 1)], 2)              # [B, J, 3, T]
    d = torch.where(w[:, :, None] != 0, p - c_t, torch.zeros_like(p))
    G = 0.5 * (w[:, :, None] * d * d).sum((1, 2, 3))
    e = w[:, :, None] * d
    gx = torch.zeros_like(x)
    gx[:, 3] = e[:, 0, 1]
    gqx, gqz = _rot(c[:, None], -s[:, None], e[:, 1:, 0], e[:, 1:, 2])
    gq = torch.stack([gqx, e[:, 1:, 1], gqz], 2)                                     # [B, J-1, 3, T]
    gx[:, 4:R] = gq.reshape(B, R - 4, T)
    gpx, gpz = e[:, :, 0].sum(1), e[:, :, 2].sum(1)
    gwx, gwz = torch.flip(torch.cumsum(torch.flip(gpx, [-1]), -1), [-1]), torch.flip(torch.cumsum(torch.flip(gpz, [-1]), -1), [-1])
    gyaw = 2 * (e[:, 1:, 2] * rx - e[:, 1:, 0] * rz).sum(1) + 2 * (gwz * wx - gwx * wz)
    if mutant == "no_yaw":
        gyaw = torch.zeros_like(gyaw)
    gvx, gvz = _rot(c, -s, gwx, gwz)
    if mutant == "vel_shift":
        gx[:, 1], gx[:, 2] = gvx, gvz
        gx[:, 1, 0] = gx[:, 2, 0] = 0
    else:
        gx[:, 1, :-1], gx[:, 2, :-1] = gvx[:, 1:], gvz[:, 1:]
    suffix = torch.flip(torch.cumsum(torch.flip(gyaw, [-1]), -1), [-1])
    gx[:, 0] = suffix - gyaw                                                          # sum over t > u
    return G, gx if mutant == "no_std" else gx * sd


def guide_manual(x0, mean, std, target, weight, step, iters, mutant=None):
    """guide() through grad_manual; mutant as there, or 'sign' (x0 <- x0 + step * grad)."""
    x = _flat(x0).clone()
    losses = []
    for k in range(iters + 1):
        G, g = grad_manual(x, mean, std, target, weight, None if mutant == "sign" else mutant)
        losses.append(G)
        if k == iters:
            break
        x = x + step * g if mutant == "sign" else x - step * g
    return x.reshape(x0.shape), torch.stack(losses)


def guided_denoiser(denoise, mean, std, target, weight, step, iters):
    """denoise(x, i) followed by the guidance of its x0 (fp64, rounded back to x0's dtype)."""
    def f(x, i):
        x0 = denoise(x, i)
        with torch.enable_grad():
            g, _ = guide(x0, mean, std, target, weight, step, iters)
        return g.to(x0.dtype)
    return f


def motion_stats(D, seed=7):
    """mean, std fp32 [D] with HumanML3D-like scales on the ric features (yaw velocity ~0.02 rad / frame, root velocity
    ~0.03 m / frame, height ~0.9 m, joints within ~0.5 m of the root) and the synthetic stand-in elsewhere."""
    g = torch.Generator().manual_seed(seed)
    R = ric_features(n_joints(D))
    mean, std = torch.randn(D, generator=g) * 0.3, 0.2 + 1.8 * torch.rand(D, generator=g)
    mean[:4] = torch.tensor([0.0, 0.0, 0.03, 0.9])
    std[:4] = torch.tensor([0.02, 0.03, 0.03, 0.1])
    mean[4:R] = (torch.rand(R - 4, generator=g) - 0.5)
    std[4:R] = 0.05 + 0.1 * torch.rand(R - 4, generator=g)
    return mean, std


def step_bound(std, weight, extent, T):
    """The step size the tests use, 1 / L_GN (DESIGN.md, "Joint-position control"): L_GN = s^2 W (1 + T (1 + 4 A^2)) bounds
    the Gauss-Newton part of the Hessian of G in normalised units, with s = max std of the ric features, W = the largest
    per-sample sum of the weights and A = `extent`, a bound on the XZ distance of a weighted joint from an earlier root
    position (metres)."""
    R = ric_features(n_joints(std.shape[0]))
    s2 = float(std[:R].double().max()) ** 2
    W = float(weight.double().sum((1, 2)).max())
    return 1.0 / (s2 * W * (1 + T * (1 + 4 * extent ** 2)))
