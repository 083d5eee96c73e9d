"""TEST INFRASTRUCTURE ONLY -- the handshake of chained windows (this project's definition, DESIGN.md "Long motions
from chained windows") as a plain torch wrapper around any denoiser, so that the UNMODIFIED reference sampler can run it
(oracle/gen_golden_handshake.py) and the fp32 oracles of this directory can follow it.

Window b (a batch sample) has n_b = y['lengths'][b] frames (all T without lengths); y['motion_start'][b] marks the
windows that begin a motion (absent: the whole batch is one motion).  For a window b that does not, p = b - 1 and
j = 0 .. h-1, both D[p, ..., n_p - h + j] and D[b, ..., j] become

    H_j = (1 - a_j) * D[p, ..., n_p - h + j] + a_j * D[b, ..., j],   a_j = (j + 1) / (h + 1)

(a_j rounded once to the dtype of D).  D is the wrapped model's output, read before any frame is replaced.
"""
import numpy as np
import torch
import torch.nn as nn


def pairs(batch, nframes, h, lengths=None, motion_start=None):
    """[(p, b, n_p)] for every window b that continues window p = b - 1."""
    n = [nframes] * batch if lengths is None else [int(v) for v in torch.as_tensor(lengths).reshape(-1)]
    ms = [True] + [False] * (batch - 1) if motion_start is None else [bool(v) for v in torch.as_tensor(motion_start).reshape(-1)]
    assert ms[0]
    return [(b - 1, b, n[b - 1]) for b in range(1, batch) if not ms[b]] if h > 0 else []


def blend(D, h, lengths=None, motion_start=None, alpha_reversed=False, suffix_shift=0, ignore_motion_start=False):
    """The handshake applied to D [B, ..., T].  The keywords make the mutants the kernel tests must tell apart:
    alpha_reversed uses a_{h-1-j}; suffix_shift moves the suffix frame by that many; ignore_motion_start chains
    every window to its predecessor."""
    B, T = D.shape[0], D.shape[-1]
    out = D.clone()
    for p, b, n_p in pairs(B, T, h, lengths, None if ignore_motion_start else motion_start):
        for j in range(h):
            jj = h - 1 - j if alpha_reversed else j
            a = torch.tensor((jj + 1) / (h + 1), dtype=D.dtype)
            fp = n_p - h + j + suffix_shift
            v = (1 - a) * D[p, ..., fp] + a * D[b, ..., j]
            out[p, ..., fp] = v
            out[b, ..., j] = v
    return out


def blend_np(D, h, lengths, motion_start):
    """A direct numpy restatement of `blend` in fp64, loop by loop, for the oracle's own test."""
    D = np.asarray(D, dtype=np.float64)
    out = D.copy()
    for b in range(1, D.shape[0]):
        if motion_start[b]:
            continue
        n_p = lengths[b - 1]
        for j in range(h):
            a = (j + 1.0) / (h + 1.0)
            v = (1.0 - a) * D[b - 1, ..., n_p - h + j] + a * D[b, ..., j]
            out[b - 1, ..., n_p - h + j] = v
            out[b, ..., j] = v
    return out


class HandshakeWrapper(nn.Module):
    """model(x, t, y=y) followed by `blend` on y['lengths'] / y['motion_start']: the reference's sampler sees the blend
    as part of the model output, ahead of inpainting and clip_denoised (gaussian_diffusion.py:298-304)."""

    def __init__(self, model, h):
        super().__init__()
        self.model = model
        self.h = int(h)

    def forward(self, x, timesteps, y=None, **kw):
        out = self.model(x, timesteps, y=y, **kw)
        y = y or {}
        return blend(out, self.h, y.get("lengths"), y.get("motion_start"))

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self._modules["model"], name)


def denoiser(denoise, h, lengths, motion_start):
    """denoise(x, i) -> x0 followed by the blend: the interface of oracle/plms_oracle.py and oracle/dpm_oracle.py."""
    return lambda x, i: blend(denoise(x, i), h, lengths, motion_start)
