"""TEST INFRASTRUCTURE ONLY -- refined transitions between chained windows (DoubleTake's second take; this project's
definition, DESIGN.md "Refined transitions") as plain torch, so that the UNMODIFIED reference sampler can run them
(oracle/gen_golden_double_take.py) and the fp32 oracles of this directory can follow them.

Soft inpainting of x0 with weight w (1 = keep the motion):  w >= 1 -> motion;  w <= 0 -> x0;  otherwise
(1 - w) * x0 + w * motion in the dtype of x0, each operation rounded.  `SoftInpaintWrapper` applies it to the model
output, where the reference's sampler applies the bool mask (gaussian_diffusion.py:298-304): ahead of clip_denoised.

A transition between window p and the window b = p + 1 that continues it has Lt = 2m + h frames: p's frames
n_p - h - m .. n_p - 1, then b's frames h .. h + m - 1, with weights (m - f)/m for f < m, 0 over the handshake and
(f - m - h + 1)/m after it.  Its frames 1 .. Lt - 2 replace frames [s - m + 1, s + h + m - 1) of the stitched motion, s the
frame where b's handshake begins in it.
"""
import numpy as np
import torch
import torch.nn as nn


def soft_inpaint(x0, w, motion, swap=False, clamp_first=False, clip=False):
    """The blend of x0 [B, ...] in x0's dtype, then the clamp when `clip`.  Mutants for the kernel tests: swap exchanges
    w and 1 - w; clamp_first clamps before the blend."""
    if clip and clamp_first:
        x0 = x0.clamp(-1, 1)
    a, c = (w, 1 - w) if swap else (1 - w, w)
    out = torch.where(w >= 1, motion, torch.where(w <= 0, x0, a * x0 + c * motion))
    if clip and not clamp_first:
        out = out.clamp(-1, 1)
    return out


def soft_inpaint_np(x0, w, motion):
    """fp64 numpy restatement of soft_inpaint, element by element."""
    x0, w, motion = (np.asarray(v, dtype=np.float64) for v in (x0, w, motion))
    out = np.empty_like(x0)
    for i in np.ndindex(x0.shape):
        out[i] = motion[i] if w[i] >= 1 else x0[i] if w[i] <= 0 else (1 - w[i]) * x0[i] + w[i] * motion[i]
    return out


class SoftInpaintWrapper(nn.Module):
    """model(x, t, y=y) followed by soft_inpaint with y['inpainting_weight'] / y['inpainted_motion'] (when present).  A y
    without 'inpainting_mask' leaves the reference's own inpainting off, so the sampler sees only this blend."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x, timesteps, y=None, **kw):
        out = self.model(x, timesteps, y=y, **kw)
        y = y or {}
        if "inpainting_weight" in y:
            out = soft_inpaint(out, y["inpainting_weight"].to(out.dtype), y["inpainted_motion"].to(out.dtype))
        return out

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self._modules["model"], name)


def denoiser(denoise, weight, motion):
    """denoise(x, i) -> x0 followed by the soft blend: the interface of oracle/plms_oracle.py and oracle/dpm_oracle.py."""
    return lambda x, i: soft_inpaint(denoise(x, i), weight.to(torch.float32), motion.to(torch.float32))


def weights(h, m):
    """[Lt] fp32, each weight in fp64 rounded once."""
    Lt = 2 * m + h
    w = [(m - f) / m if f < m else 0.0 if f < m + h else (f - m - h + 1) / m for f in range(Lt)]
    return torch.tensor(w, dtype=torch.float64).float()


def layout(lengths, motion_start, h, m):
    """[(p, b, motion index, s)] per transition; s = where b's handshake begins in the stitched motion."""
    n = [int(v) for v in lengths]
    out, k, off = [], -1, [0] * len(n)
    for b, start in enumerate(motion_start):
        if start:
            k += 1
            continue
        off[b] = off[b - 1] + n[b - 1] - h
        out.append((b - 1, b, k, off[b]))
    return out


def gather(windows, lengths, motion_start, h, m):
    """x_init [n, J, F, Lt] of every transition, frame by frame."""
    rows = []
    for p, b, _, _ in layout(lengths, motion_start, h, m):
        n_p = int(lengths[p])
        frames = [windows[p, ..., n_p - h - m + f] for f in range(m + h)] + [windows[b, ..., f - m] for f in range(m + h, 2 * m + h)]
        rows.append(torch.stack(frames, dim=-1))
    return torch.stack(rows)


def stitch(windows, lengths, motion_start, h):
    """The motions of the windows: the first window's [:n], then each later window's [h:n]."""
    motions = []
    for b in range(windows.shape[0]):
        n = int(lengths[b])
        if motion_start[b]:
            motions.append([windows[b, ..., :n]])
        else:
            motions[-1].append(windows[b, ..., h:n])
    return [torch.cat(p, dim=-1) for p in motions]


def paste(motions, refined, lengths, motion_start, h, m):
    """Copies of the motions with frames 1 .. Lt - 2 of each refined transition pasted in."""
    out = [x.clone() for x in motions]
    Lt = 2 * m + h
    for i, (_, _, k, s) in enumerate(layout(lengths, motion_start, h, m)):
        for f in range(1, Lt - 1):
            out[k][..., s - m + f] = refined[i, ..., f]
    return out


def transition_y(y, lengths, motion_start, h, m, x_init):
    """y of the transition batch: window b's text_embed and scale, all frames valid, the soft weights and x_init."""
    bs = [b for _, b, _, _ in layout(lengths, motion_start, h, m)]
    n, Lt = len(bs), 2 * m + h
    J, F = x_init.shape[1], x_init.shape[2]
    out = dict(mask=torch.ones((n, 1, 1, Lt), dtype=torch.bool), lengths=torch.full((n,), Lt, dtype=torch.long),
               inpainting_weight=weights(h, m).view(1, 1, 1, Lt).expand(n, J, F, Lt).contiguous(), inpainted_motion=x_init)
    te = y["text_embed"]
    out["text_embed"] = te if te.shape[1] == 1 else te[:, bs]
    if "scale" in y:
        out["scale"] = y["scale"][bs]
    return out
