"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

fp64 statement of goal-directed autoregressive chains (DESIGN.md, "Goals in the world frame").  W is the frame of
recover_from_ric on the returned motion; chunk c starts at frame g_c of it.  recover_root_rot_pos (oracle/ric_oracle.py)
over the whole returned motion, read at frame g_c, gives the quaternion (cos yaw_c, 0, sin yaw_c, 0) and the root
position P_c, and

    recover_from_ric(returned)[g_c + t] = M_c(recover_from_ric(chunk c alone)[t]),   M_c = qrot(qinv(q_c), .) then + P_c in XZ

so a goal in W is chunk c's target M_c^-1(goal): XZ translated by -P_c and rotated by qrot(q_c, .), y unchanged.
recover_root_rot_heading_ang's heading atan2(forward.x, forward.z) turns under M_c by delta_c = the atan2(x, z) angle of
M_c applied to (0, 0, 1), so the heading entry becomes wrap(heading - delta_c) into (-pi, pi].  Nothing here uses the
engine's carry recurrence: every frame quantity is read off the whole motion at g_c.
"""
import math

import torch

from . import ric_oracle as ro


def _denorm(motion, mean, std):
    """motion [B, D, (1,) N] normalised -> [B, N, D] fp64, de-normalised in fp32 as the reference's motion * std + mean"""
    x = motion.reshape(motion.shape[0], motion.shape[1], -1).to(torch.float32).cpu()
    data = x * std.to(torch.float32).cpu()[None, :, None] + mean.to(torch.float32).cpu()[None, :, None]
    return data.permute(0, 2, 1).double()


def frame_at(motion, mean, std, g):
    """The frame of returned frame g: dict(yaw [B], c [B], s [B], P [B, 2] (x, z)); yaw is the plain fp64 sum of the
    yaw velocities before g, c / s and P are recover_root_rot_pos's at g (g may equal the motion's length: the frame
    the next chunk would start at)."""
    data = _denorm(motion, mean, std)
    B, N, D = data.shape
    if g == N:                                   # one frame past the end: its root features do not enter frame g
        data = torch.cat([data, torch.zeros(B, 1, D, dtype=data.dtype)], dim=1)
    c, s, pos = ro.recover_root_rot_pos(data[:, :g + 1])
    yaw = data[:, :g, 0].sum(dim=1)
    return dict(yaw=yaw, c=c[:, g], s=s[:, g], P=pos[:, g][:, [0, 2]])


def carry_after(motion, mean, std, n):
    """The engine's carry after frames 0 .. n-1, read off the motion: [B, 6] fp64 (yaw = sum of the first n yaw
    velocities, P = root XZ at frame n-1, the root XZ velocity of frame n-1, 1.0 when n > 0)."""
    data = _denorm(motion, mean, std)
    B = data.shape[0]
    out = torch.zeros(B, 6, dtype=torch.float64)
    if n == 0:
        return out
    _, _, pos = ro.recover_root_rot_pos(data[:, :n])
    out[:, 0] = data[:, :n, 0].sum(dim=1)
    out[:, 1], out[:, 2] = pos[:, n - 1, 0], pos[:, n - 1, 2]
    out[:, 3], out[:, 4] = data[:, n - 1, 1], data[:, n - 1, 2]
    out[:, 5] = 1.0
    return out


def wrap(h):
    """into (-pi, pi], as atan2 returns"""
    return h - 2 * math.pi * torch.ceil((h - math.pi) / (2 * math.pi))


def to_chunk(goal, fr):
    """goal [B, n_ext, 3] in W -> fp64 target in the chunk frame fr (frame_at); the last entry is the heading."""
    goal = goal.double().cpu()
    out = goal.clone()
    c, s = fr["c"][:, None], fr["s"][:, None]
    d = torch.stack([goal[:, :-1, 0] - fr["P"][:, 0:1], torch.zeros_like(goal[:, :-1, 0]), goal[:, :-1, 2] - fr["P"][:, 1:2]], -1)
    loc = ro._rot_y_inv(c, -s, d)                # qrot(q, .) = qrot(qinv(qinv(q)), .)
    out[:, :-1, 0], out[:, :-1, 2] = loc[..., 0], loc[..., 2]
    fwd = ro._rot_y_inv(fr["c"], fr["s"], torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(goal.shape[0], 3))
    delta = torch.atan2(fwd[:, 0], fwd[:, 2])
    out[:, -1, 0] = wrap(goal[:, -1, 0] - delta)
    return out


def to_world(target, fr):
    """The inverse of to_chunk: a chunk-frame target [B, n_ext, 3] -> W."""
    t = target.double().cpu()
    out = t.clone()
    d = torch.stack([t[:, :-1, 0], torch.zeros_like(t[:, :-1, 0]), t[:, :-1, 2]], -1)
    w = ro._rot_y_inv(fr["c"][:, None], fr["s"][:, None], d)
    out[:, :-1, 0], out[:, :-1, 2] = w[..., 0] + fr["P"][:, 0:1], w[..., 2] + fr["P"][:, 1:2]
    fwd = ro._rot_y_inv(fr["c"], fr["s"], torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(t.shape[0], 3))
    out[:, -1, 0] = wrap(t[:, -1, 0] + torch.atan2(fwd[:, 0], fwd[:, 2]))
    return out


def chunk_targets(returned, mean, std, goals, off, pred_len, n_chunks):
    """Every chunk's target [n_chunks, B, n_ext, 3] fp64: goals [n_goals, B, n_ext, 3] (n_goals 1 or n_chunks) mapped
    into the frame of g_c = off + c * pred_len of the returned motion [B, D, (1,) >= g_{n-1}]."""
    out = []
    for c in range(n_chunks):
        fr = frame_at(returned, mean, std, off + c * pred_len)
        out.append(to_chunk(goals[0 if goals.shape[0] == 1 else c], fr))
    return torch.stack(out)
