"""TEST INFRASTRUCTURE ONLY -- plain-torch restatement of the reference's variational bound (diffusion/gaussian_diffusion.py
:1189-1222 _vb_terms_bpd, :1527-1599 _prior_bpd / calc_bpd_loop; diffusion/losses.py), on top of the denoisers of
oracle/plms_oracle.py.  Pinned against the live reference by tests/golden/vb_small.npz (oracle/gen_golden_vb.py).

fp32 (`dtype=torch.float32`, the default) follows the reference's operation order on its fp32 tables; fp64 runs the
same formulas on the fp64 tables (the conditioning yardstick of the t = 0 decoder term, DESIGN.md section 1).  The
engine's own reduction order (per 32-column chunk, then the 256-lane block sum of vb_reduce_kernel) is restated by
`engine_mean` for the bit-exact epilogue tests.
"""
import math

import numpy as np
import torch

from . import mdm_oracle as mo
from . import plms_oracle as po


def model_log_variance(tables, var_type="small"):
    """p_mean_variance's fixed log-variance (gaussian_diffusion.py:325-345): 'small' or 'large'."""
    if var_type == "small":
        return tables["posterior_log_variance_clipped"]
    return np.log(np.append(tables["posterior_variance"][1], tables["betas"][1:]))


def normal_kl(mean1, logvar1, mean2, logvar2):
    """losses.py:12-39 in its operation order."""
    return 0.5 * (-1.0 + logvar2 - logvar1 + torch.exp(logvar1 - logvar2) + ((mean1 - mean2) ** 2) * torch.exp(-logvar2))


def approx_standard_normal_cdf(x):
    """losses.py:42-47."""
    return 0.5 * (1.0 + torch.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * torch.pow(x, 3))))


def discretized_gaussian_log_likelihood(x, means, log_scales):
    """losses.py:50-77."""
    centered_x = x - means
    inv_stdv = torch.exp(-log_scales)
    cdf_plus = approx_standard_normal_cdf(inv_stdv * (centered_x + 1.0 / 255.0))
    cdf_min = approx_standard_normal_cdf(inv_stdv * (centered_x - 1.0 / 255.0))
    log_cdf_plus = torch.log(cdf_plus.clamp(min=1e-12))
    log_one_minus_cdf_min = torch.log((1.0 - cdf_min).clamp(min=1e-12))
    cdf_delta = cdf_plus - cdf_min
    return torch.where(x < -0.999, log_cdf_plus,
                       torch.where(x > 0.999, log_one_minus_cdf_min, torch.log(cdf_delta.clamp(min=1e-12))))


def mean_flat(t):
    return t.mean(dim=list(range(1, t.dim())))


def _tab(tables, key, i, dtype):
    """_extract_into_tensor: table[i] as an fp32 scalar (fp64 for the fp64 restatement); key: a table name or array."""
    arr = tables[key] if isinstance(key, str) else key
    return mo.f32(arr, i) if dtype == torch.float32 else torch.tensor(float(arr[i]), dtype=dtype)


def vb_terms(tables, x_start, x_t, i, x0, noise, var_type="small", dtype=torch.float32):
    """Per-element (term, (x0 - x_start)^2, (eps - noise)^2) of schedule index i; x0 after inpainting and clamp.  term is
    normal_kl in nats, or at i == 0 the decoder NLL in nats (not yet averaged, not yet in bits)."""
    x_start, x_t, x0, noise = (v.to(dtype) for v in (x_start, x_t, x0, noise))
    g = lambda key: _tab(tables, key, i, dtype)  # noqa: E731
    lvm = g(model_log_variance(tables, var_type))
    c1, c2 = g("posterior_mean_coef1"), g("posterior_mean_coef2")
    mean = c1 * x0 + c2 * x_t
    if i == 0:
        term = -discretized_gaussian_log_likelihood(x_start, mean, 0.5 * lvm)
    else:
        true_mean = c1 * x_start + c2 * x_t
        term = normal_kl(true_mean, g("posterior_log_variance_clipped"), mean, lvm)
    eps = (g("sqrt_recip_alphas_cumprod") * x_t - x0) / g("sqrt_recipm1_alphas_cumprod")
    return term, (x0 - x_start) ** 2, (eps - noise) ** 2


def prior_bpd(tables, x_start, dtype=torch.float32):
    """_prior_bpd (gaussian_diffusion.py:1527-1542)."""
    n = len(tables["betas"])
    x_start = x_start.to(dtype)
    mean = _tab(tables, "sqrt_alphas_cumprod", n - 1, dtype) * x_start
    lv = _tab(tables, "log_one_minus_alphas_cumprod", n - 1, dtype)
    return mean_flat(normal_kl(mean, lv, torch.zeros((), dtype=dtype), torch.zeros((), dtype=dtype))) / np.log(2.0)


def vb_loop(denoise, tables, x_start, tape, clip_denoised=True, inpaint=None, var_type="small", dtype=torch.float32):
    """calc_bpd_loop with an explicit noise tape [eps_{n-1}, ..., eps_0] and denoise(x, i) -> model output (CFG included).
    Returns the reference's dict; dtype float64 runs the bound arithmetic (not the denoiser) in fp64."""
    n = len(tables["betas"])
    vb, xm, em = [], [], []
    for k, i in enumerate(range(n)[::-1]):
        noise = tape[k]
        x_t = mo.q_sample(tables, x_start, i, noise)
        x0 = po.p_mean_x0(denoise(x_t, i), clip_denoised, inpaint)
        term, xe, ee = vb_terms(tables, x_start, x_t, i, x0, noise, var_type, dtype)
        vb.append(mean_flat(term) / np.log(2.0))
        xm.append(mean_flat(xe))
        em.append(mean_flat(ee))
    vb, xm, em = torch.stack(vb, 1), torch.stack(xm, 1), torch.stack(em, 1)
    prior = prior_bpd(tables, x_start, dtype)
    return {"total_bpd": vb.sum(1) + prior, "prior_bpd": prior, "vb": vb, "xstart_mse": xm, "mse": em}


# ---------------------------------------------------------------------------------------------------------------------
# The engine's reduction order (csrc/epilogues.cuh OutVb, csrc/kernels.cuh vb_reduce_kernel / vb_block_sum), fp32
LANES = 256


def block_sum(v):
    """vb_block_sum over the last axis of v (fp32): lane k adds v[k], v[k + 256], ... in order, then the tree
    s = 128, 64, ..., 1 of sh[k] += sh[k + s]."""
    v = v.to(torch.float32)
    n = v.shape[-1]
    m = (n + LANES - 1) // LANES
    pad = torch.zeros(v.shape[:-1] + (m * LANES - n,), dtype=torch.float32, device=v.device)
    rows = torch.cat([v, pad], -1).reshape(v.shape[:-1] + (m, LANES))
    acc = torch.zeros(v.shape[:-1] + (LANES,), dtype=torch.float32, device=v.device)
    for r in range(m):
        acc = acc + rows[..., r, :]
    s = LANES // 2
    while s > 0:
        acc = torch.cat([acc[..., :s] + acc[..., s:2 * s], acc[..., s:]], -1)
        s //= 2
    return acc[..., 0]


def chunk_sums(elem, drop_last_chunk=False):
    """elem [B, J, T] fp32 -> the epilogue's partial sums [B, T, ceil(J/32)]: columns 32c .. 32c + 31 added in order,
    starting from 0."""
    B, J, T = elem.shape
    nc = (J + 31) // 32
    out = torch.zeros((B, T, nc), dtype=torch.float32, device=elem.device)
    for c in range(nc):
        if drop_last_chunk and c == nc - 1:
            continue
        s = torch.zeros((B, T), dtype=torch.float32, device=elem.device)
        for j in range(32 * c, min(J, 32 * c + 32)):
            s = s + elem[:, j, :]
        out[:, :, c] = s
    return out


def engine_mean(elem, bits=False, drop_last_chunk=False):
    """The per-sample mean of vb_reduce_kernel: elem [B, J, F, T] (or [B, J, T]) fp32 -> [B]."""
    B, T = elem.shape[0], elem.shape[-1]
    e = elem.reshape(B, -1, T).to(torch.float32)
    J = e.shape[1]
    s = block_sum(chunk_sums(e, drop_last_chunk).reshape(B, -1))
    m = s / torch.tensor(float(J * T), dtype=torch.float32)
    if bits:
        m = m / torch.tensor(np.float32(math.log(2.0)))
    return m
