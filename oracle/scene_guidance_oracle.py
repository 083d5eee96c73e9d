"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

fp64 restatement of the scene terms of joint-position control (DESIGN.md, "Joint-position control", "Scene: obstacles
and uneven ground"):

    G = G_joint + G_contact + 1/2 lf sum_{t<L, j} min(p[t,j].y - h - H(p.x, p.z), 0)^2
                            + 1/2 lo sum_{t<L, j} max(r - S(p[t,j].x, p[t,j].z), 0)^2,

p = recover_from_ric(x0 * std + mean) (oracle/ric_oracle.py), G_joint and G_contact as oracle/joint_control_oracle.py and
oracle/foot_guidance_oracle.py state them, S (the obstacles' signed distance) and H (the terrain) bilinear samples of
b200mdm.SceneGrid grids as DESIGN.md defines them.

`guide` takes the gradient with torch.autograd; `grad_manual` writes the scene terms' position adjoint e out and hands it
to joint_control_oracle.grad_manual's chain (the joint and contact terms' gradient is foot_guidance_oracle.grad_manual's),
with optional mutants for the tests' sensitivity checks.  `guided_denoiser` wraps a denoise(x, i) of the oracles as
joint_control_oracle's does.
"""
import torch

from . import foot_guidance_oracle as fo
from . import joint_control_oracle as jo

# u and v swapped; the grids' gradient's sign flipped; the margin's sign flipped; clamping ignored (the edge cells
# extrapolated); sample b reading grid b + 1; dH dropped from x / z (the terrain acting in y only)
MUTANTS = ("swap_uv", "grad_sign", "margin_sign", "no_clamp", "grid_shift", "terrain_y_only")


def sample(grid, x, z, mutant=None):
    """(value, d/dx, d/dz) fp64 [B, N] of a SceneGrid at x, z [B, N] (the value differentiable in x and z): the bilinear
    interpolant of cell (min(floor(v), Gz - 2), min(floor(u), Gx - 2)) at the clamped u, v, its gradient 0 along a
    clamped axis."""
    B = x.shape[0]
    V = grid.values.double()
    V = (V if grid.per_sample else V.expand(B, -1, -1)).reshape(B, -1)
    if mutant == "grid_shift":
        V = torch.roll(V, -1, 0)
    gz, gx = grid.shape
    if mutant == "swap_uv":
        x, z = z, x
    c = grid.cell
    ur, vr = (x - grid.origin[0]) / c, (z - grid.origin[1]) / c
    if mutant == "no_clamp":
        u, v = ur, vr
        inu = inv = torch.ones_like(ur)
    else:
        u, v = ur.clamp(0, gx - 1), vr.clamp(0, gz - 1)
        inu, inv = ((ur >= 0) & (ur <= gx - 1)).double(), ((vr >= 0) & (vr <= gz - 1)).double()
    k = torch.floor(u.detach()).clamp(0, gx - 2).long()
    i = torch.floor(v.detach()).clamp(0, gz - 2).long()
    a, b = u - k, v - i
    idx = i * gx + k
    v00, v01, v10, v11 = (torch.gather(V, 1, idx + o) for o in (0, 1, gx, gx + 1))
    val = (1 - b) * ((1 - a) * v00 + a * v01) + b * ((1 - a) * v10 + a * v11)
    dx = ((1 - b.detach()) * (v01 - v00) + b.detach() * (v11 - v10)) / c * inu
    dz = ((1 - a.detach()) * (v10 - v00) + a.detach() * (v11 - v01)) / c * inv
    return val, dx, dz


def _live(lengths, B, T):
    return (torch.arange(T)[None, :] < fo._lengths(lengths, B, T)[:, None]).double()     # [B, T]


def scene_terms(x0, mean, std, floor_w, floor_h, obstacle_w, margin, sdf=None, terrain=None, lengths=None):
    """(floor energy over the terrain [B], obstacle energy [B]) of normalised x0 [B, D, T] (fp64, differentiable)."""
    B, D, T = x0.shape
    p = fo._positions(x0, mean, std).reshape(B, -1, 3)                                 # [B, T * J, 3]
    J = p.shape[1] // T
    live = _live(lengths, B, T).repeat_interleave(J, 1)                                 # [B, T * J]
    zero = torch.zeros(B, dtype=torch.float64)
    ef = eo = zero
    if floor_w > 0:
        H = sample(terrain, p[..., 0], p[..., 2])[0] if terrain is not None else 0.0
        m = torch.clamp(p[..., 1] - floor_h - H, max=0.0)
        ef = 0.5 * floor_w * (live * m * m).sum(1)
    if obstacle_w > 0:
        m = torch.clamp(margin - sample(sdf, p[..., 0], p[..., 2])[0], min=0.0)
        eo = 0.5 * obstacle_w * (live * m * m).sum(1)
    return ef, eo


def loss(x0, mean, std, target, weight, contact_w, floor_w, floor_h, obstacle_w, margin, sdf, terrain, kappa, lengths=None):
    """total G per sample [B] of x0 [B, D, T] (fp64, differentiable) with a fixed kappa [B, 4, T]"""
    ec, _ = fo.foot_terms(x0, mean, std, kappa, contact_w, 0.0, floor_h, lengths)
    ef, eo = scene_terms(x0, mean, std, floor_w, floor_h, obstacle_w, margin, sdf, terrain, lengths)
    return jo.loss(x0, mean, std, target, weight) + ec + ef + eo


def guide(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h, obstacle_w, margin, sdf=None,
          terrain=None, contact=None, lengths=None):
    """(guided x0 fp64 in x0's shape, total G fp64 [iters + 1, B]) by autograd; kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = fo._kappa(x0, mean, std, contact, lengths)
    losses = []
    for k in range(iters + 1):
        x.requires_grad_(True)
        G = loss(x, mean, std, target, weight, contact_w, floor_w, floor_h, obstacle_w, margin, sdf, terrain, kappa, lengths)
        losses.append(G.detach())
        if k == iters:
            break
        (g,) = torch.autograd.grad(G.sum(), x)
        x = (x - step * g).detach()
    return x.detach().reshape(x0.shape), torch.stack(losses)


def grad_manual(x0, mean, std, target, weight, contact_w, floor_w, floor_h, obstacle_w, margin, sdf=None, terrain=None,
                contact=None, lengths=None, mutant=None, kappa=None):
    """(G [B], dG/dx0 [B, D, T]) in fp64: the scene terms' position adjoint of DESIGN.md,
    e.x += -lo m_o dS/dx - lf m_f dH/dx (and in z), e.y += lf m_f with m_o = max(r - S, 0), m_f = min(p.y - h - H, 0),
    through joint_control_oracle.grad_manual's chain, plus the joint and contact terms of foot_guidance_oracle.grad_manual.
    mutant: None or one of MUTANTS."""
    x0 = jo._flat(x0)
    B, D, T = x0.shape
    J = jo.n_joints(D)
    if kappa is None:
        kappa = fo._kappa(x0, mean, std, contact, lengths)
    G, g = fo.grad_manual(x0, mean, std, target, weight, contact_w, 0.0, floor_h, contact, lengths, kappa=kappa)
    p = fo._positions(x0, mean, std)                                                     # [B, T, J, 3]
    px, py, pz = (p[..., a].reshape(B, T * J) for a in range(3))
    live = _live(lengths, B, T).repeat_interleave(J, 1)
    e = torch.zeros(B, T * J, 3, dtype=torch.float64)
    sign = -1.0 if mutant == "grad_sign" else 1.0
    if floor_w > 0:
        H, hx, hz = sample(terrain, px, pz, mutant) if terrain is not None else (0.0, 0.0, 0.0)
        m = live * torch.clamp(py - floor_h - H, max=0.0)
        e[..., 1] += floor_w * m
        if mutant != "terrain_y_only":
            e[..., 0] -= sign * floor_w * m * hx
            e[..., 2] -= sign * floor_w * m * hz
        G = G + 0.5 * floor_w * (m * m).sum(1)
    if obstacle_w > 0:
        S, sx, sz = sample(sdf, px, pz, mutant)
        m = live * torch.clamp((-margin if mutant == "margin_sign" else margin) - S, min=0.0)
        e[..., 0] -= sign * obstacle_w * m * sx
        e[..., 2] -= sign * obstacle_w * m * sz
        G = G + 0.5 * obstacle_w * (m * m).sum(1)
    e = e.reshape(B, T, J, 3).permute(0, 2, 3, 1)                                         # [B, J, 3, T]
    pj = p.permute(0, 2, 3, 1)
    _, gs = jo.grad_manual(x0, mean, std, pj - e, torch.ones(B, J, T, dtype=torch.float64))
    return G, g + gs


def guide_manual(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h, obstacle_w, margin, sdf=None,
                 terrain=None, contact=None, lengths=None, mutant=None):
    """guide() through grad_manual; mutant as there.  kappa is read once, from x0."""
    x = jo._flat(x0).clone()
    kappa = fo._kappa(x0, mean, std, contact, lengths)
    losses = []
    for k in range(iters + 1):
        G, g = grad_manual(x, mean, std, target, weight, contact_w, floor_w, floor_h, obstacle_w, margin, sdf, terrain,
                           contact, lengths, mutant, kappa)
        losses.append(G)
        if k == iters:
            break
        x = x - step * g
    return x.reshape(x0.shape), torch.stack(losses)


def guided_denoiser(denoise, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h, obstacle_w, margin,
                    sdf=None, terrain=None, contact=None, lengths=None):
    """denoise(x, i) followed by the guidance of its x0 (fp64, rounded back to x0's dtype)."""
    def f(x, i):
        x0 = denoise(x, i)
        with torch.enable_grad():
            g, _ = guide(x0, mean, std, target, weight, step, iters, contact_w, floor_w, floor_h, obstacle_w, margin, sdf,
                         terrain, contact, lengths)
        return g.to(x0.dtype)
    return f


def max_slope(grid):
    """the grid's largest finite-difference slope |V[i, k+1] - V[i, k]| / cell or |V[i+1, k] - V[i, k]| / cell"""
    V = grid.values.double()
    return float(max((V[..., :, 1:] - V[..., :, :-1]).abs().max(), (V[..., 1:, :] - V[..., :-1, :]).abs().max())) / grid.cell


def step_bound(std, weight, extent, T, contact_w, floor_w, obstacle_w, sdf=None, terrain=None, kappa_max=1.0):
    """The step size the tests use, 1 / L_GN with the scene terms (DESIGN.md, "Scene: obstacles and uneven ground"):
    L_GN = s^2 (W g + 4 lc kappa_max (3 + 4 A^2) + lf' + 2 lo s_S^2 J T g), g = 1 + T (1 + 4 A^2), with
    lf' = lf without a terrain and 2 lf (1 + 2 s_H^2 J T g) with one, s, W and A as in joint_control_oracle.step_bound
    and s_S, s_H the grids' largest slopes (max_slope)."""
    J = jo.n_joints(std.shape[0])
    R = jo.ric_features(J)
    s2 = float(std[:R].double().max()) ** 2
    W = float(weight.double().sum((1, 2)).max())
    gain = 1 + T * (1 + 4 * extent ** 2)
    lf = floor_w if terrain is None else 2 * floor_w * (1 + 2 * max_slope(terrain) ** 2 * J * T * gain)
    lo = 0.0 if sdf is None else 2 * obstacle_w * max_slope(sdf) ** 2 * J * T * gain
    return 1.0 / (s2 * (W * gain + 4 * contact_w * kappa_max * (3 + 4 * extent ** 2) + lf + lo))
