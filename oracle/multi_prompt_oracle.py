"""TEST INFRASTRUCTURE ONLY -- plain-torch restatement of multi-prompt guidance (DESIGN.md, "Multi-prompt guidance"):

    x0[b, f, t] = x0_u[b, f, t] + sum_{k=0..K-1} w[b, k, f, t] * (x0_k[b, f, t] - x0_u[b, f, t]),

each x0_k the denoiser under prompt k and x0_u under the empty condition (mask_cond force_mask, as
ClassifierFreeSampleModel forms its unconditional half), k ascending, one rounding per operation.  `compose` runs in the
dtype of the predictions it is given: fp32 for parity with the engine, fp64 for error bounds.

The denoisers here have the interface denoise(x, i) at schedule index i (the model timestep is timestep_map[i]; i = -1
wraps, as PLMS needs) of dec_emb_oracle.sample_loop (DDPM / DDIM), plms_oracle.plms_loop, dpm_oracle.dpm_loop and
reverse_oracle.reverse_loop.
"""
import torch

from . import dec_emb_oracle as de
from . import mdm_oracle as mo


def compose(x0_u, x0_k, w):
    """x0_u [B, J, F, T]; x0_k a list of K such tensors; w [B, K, D or 1, T or 1] with D = J * F (broadcast)."""
    B, J, Fe, T = x0_u.shape
    w = w.to(x0_u.dtype)
    x0 = x0_u.reshape(B, J * Fe, T).clone()
    u = x0.clone()
    for k, xk in enumerate(x0_k):
        x0 = x0 + w[:, k] * (xk.reshape(B, J * Fe, T) - u)
    return x0.reshape(B, J, Fe, T)


def enc_denoiser(W, timestep_map, prompts, weight, lengths=None, mask_frames=True, actions=None, cast=None):
    """trans_enc: prompts [K, B, C] text features (text models, None for action models), actions [B, K] (action
    models, None for text models), weight [B, K, D or 1, T or 1]."""
    K = int(weight.shape[1])

    def f(x, i):
        tm = int(timestep_map[i])
        if actions is not None:
            a = torch.as_tensor(actions)
            xk = [mo.denoise_enc(W, x, tm, None, lengths, mask_frames, False, a[:, k:k + 1], cast) for k in range(K)]
            xu = mo.denoise_enc(W, x, tm, None, lengths, mask_frames, True, a[:, :1], cast)
        else:
            xk = [mo.denoise_enc(W, x, tm, prompts[k:k + 1], lengths, mask_frames, False, None, cast) for k in range(K)]
            xu = mo.denoise_enc(W, x, tm, prompts[:1], lengths, mask_frames, True, None, cast)
        return compose(xu, xk, weight)
    return f


def dec_emb_denoiser(W, timestep_map, prompts, weight, lengths=None, mask_frames=True, g=None, cast=None):
    """The CLIP decoder with a timestep token: prompts [K, B, 512], g [B, d] target embedding or None (every group
    carries it)."""
    K = int(weight.shape[1])

    def f(x, i):
        tm = int(timestep_map[i])
        xk = [de.denoise_dec_emb(W, x, tm, prompts[k:k + 1], lengths, mask_frames, False, g, cast) for k in range(K)]
        xu = de.denoise_dec_emb(W, x, tm, prompts[:1], lengths, mask_frames, True, g, cast)
        return compose(xu, xk, weight)
    return f
