"""TEST INFRASTRUCTURE ONLY -- plain-torch fp32 restatement of the reference's pseudo linear multistep sampler
(diffusion/gaussian_diffusion.py:992-1187: plms_sample, plms_sample_loop_progressive), on top of the denoisers of
oracle/mdm_oracle.py.  Pinned against the live reference by tests/test_plms_cpu.py and by tests/golden/plms_small.npz
(oracle/gen_golden_plms.py).

Every table value is the reference's _extract_into_tensor fp32 value (mdm_oracle.f32); index -1 (the improved-Euler
step's second forward at t = 0) wraps to the last entry, as torch indexing does in the reference.
"""
import torch

from . import mdm_oracle as mo


def p_mean_x0(x0, clip_denoised=False, inpaint=None):
    """p_mean_variance's pred_xstart for START_X (gaussian_diffusion.py:300-304, 346-352): inpainting blend, then clamp."""
    if inpaint is not None:
        m, motion = inpaint
        x0 = (x0 * ~m) + (motion * m)
    return x0.clamp(-1, 1) if clip_denoised else x0


def eps_from_x0(tables, x, i, x0):
    """_predict_eps_from_xstart (:400-404)."""
    return (mo.f32(tables["sqrt_recip_alphas_cumprod"], i) * x - x0) / mo.f32(tables["sqrt_recipm1_alphas_cumprod"], i)


def x0_from_eps(tables, x, i, eps):
    """_predict_xstart_from_eps (:381-388)."""
    return mo.f32(tables["sqrt_recip_alphas_cumprod"], i) * x - mo.f32(tables["sqrt_recipm1_alphas_cumprod"], i) * eps


def ab_combine(old_eps, order):
    """Adams-Bashforth eps' (:1054-1064) from the history, newest last."""
    cur_order = min(order, len(old_eps))
    e = old_eps
    if cur_order == 1:
        return e[-1]
    if cur_order == 2:
        return (3 * e[-1] - e[-2]) / 2
    if cur_order == 3:
        return (23 * e[-1] - 16 * e[-2] + 5 * e[-3]) / 12
    return (55 * e[-1] - 59 * e[-2] + 37 * e[-3] - 9 * e[-4]) / 24


def plms_step(denoise, tables, x, i, order, old_eps, clip_denoised=False, inpaint=None):
    """plms_sample (:992-1074).  denoise(x, i) -> model output x0 at schedule index i (the caller maps i to the model
    timestep, wrapping i = -1).  old_eps None = the first step.  Returns (sample, pred_xstart, old_eps)."""
    abp = mo.f32(tables["alphas_cumprod_prev"], i)
    sq, s1 = torch.sqrt(abp), torch.sqrt(1 - abp)
    x0 = p_mean_x0(denoise(x, i), clip_denoised, inpaint)
    eps = eps_from_x0(tables, x, i, x0)
    if order > 1 and old_eps is None:                                       # pseudo improved Euler
        old_eps = [eps]
        mean1 = x0 * sq + s1 * eps
        x0b = p_mean_x0(denoise(mean1, i - 1), clip_denoised, inpaint)
        eps2 = eps_from_x0(tables, mean1, i - 1, x0b)
        ep = (eps + eps2) / 2
    else:
        old_eps = list(old_eps) + [eps]
        ep = ab_combine(old_eps, order)
    mean = x0_from_eps(tables, x, i, ep) * sq + s1 * ep
    if len(old_eps) >= order:
        old_eps.pop(0)
    nz = 0.0 if i == 0 else 1.0
    return mean * nz + x0 * (1 - nz), x0, old_eps


def plms_loop(denoise, tables, x_T, order=2, clip_denoised=False, inpaint=None, skip_timesteps=0, init_image=None,
              collect=None):
    """plms_sample_loop_progressive (:1118-1187) from x_T; `collect` receives every step's sample."""
    n = len(tables["betas"])
    x = x_T.clone()
    idx = list(range(n - skip_timesteps))[::-1]
    if skip_timesteps and init_image is None:
        init_image = torch.zeros_like(x)
    if init_image is not None:
        x = mo.q_sample(tables, init_image, idx[0], x)
    old = None
    for i in idx:
        x, _, old = plms_step(denoise, tables, x, i, order, old, clip_denoised, inpaint)
        if collect is not None:
            collect.append(x.clone())
    return x


def enc_denoiser(W, timestep_map, cond, scale, lengths=None, mask_frames=True, cast=None):
    """denoise(x, i) for a trans_enc model, CFG-wrapped when `scale` is given."""
    def f(x, i):
        tm = int(timestep_map[i])
        if scale is None:
            return mo.denoise_enc(W, x, tm, cond, lengths, mask_frames, False, None, cast)
        return mo.cfg_denoise_enc(W, x, tm, cond, scale, lengths, mask_frames, None, cast)
    return f


def dec_denoiser(W, timestep_map, enc_text, text_mask, prefix, scale, lengths=None, mask_frames=True, cast=None):
    """denoise(x, i) for a DiP (trans_dec, prefix completion) model with CFG."""
    def f(x, i):
        return mo.cfg_denoise_dec(W, x, int(timestep_map[i]), enc_text, text_mask, prefix, scale, lengths, mask_frames, cast)
    return f
