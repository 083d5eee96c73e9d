"""TEST INFRASTRUCTURE ONLY -- plain-torch fp32 restatement of the reference's DDIM inversion step
(diffusion/gaussian_diffusion.py:838-874, ddim_reverse_sample) and of its iteration over the schedule, on top of the
denoisers of oracle/plms_oracle.py (enc_denoiser for trans_enc, dec_denoiser for the DiP decoder).  Pinned against
the live reference by tests/golden/reverse_small.npz (oracle/gen_golden_reverse.py).

Every table value is the reference's _extract_into_tensor fp32 value (mdm_oracle.f32).
"""
import torch

from . import mdm_oracle as mo
from . import plms_oracle as po


def ddim_reverse_step(tables, x0, x, i):
    """ddim_reverse_sample's update (:861-872): x at schedule index i -> x at index i + 1, from pred_xstart x0."""
    eps = po.eps_from_x0(tables, x, i, x0)
    abn = mo.f32(tables["alphas_cumprod_next"], i)
    return x0 * torch.sqrt(abn) + torch.sqrt(1 - abn) * eps


def reverse_loop(denoise, tables, x_start, first_index=0, n_steps=None, clip_denoised=False, inpaint=None,
                 collect=None):
    """ddim_reverse_sample for i = first_index ... first_index + n_steps - 1 (default: the whole schedule).
    denoise(x, i) -> model output at schedule index i.  `collect` receives (sample, pred_xstart) of every step."""
    n = len(tables["betas"])
    n_steps = n - first_index if n_steps is None else n_steps
    x = x_start.clone()
    for i in range(first_index, first_index + n_steps):
        x0 = po.p_mean_x0(denoise(x, i), clip_denoised, inpaint)
        x = ddim_reverse_step(tables, x0, x, i)
        if collect is not None:
            collect.append((x.clone(), x0.clone()))
    return x
