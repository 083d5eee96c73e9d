"""TEST INFRASTRUCTURE ONLY -- the BERT decoder's (context_len 0) restatements for the sampling extensions, built on
oracle/mdm_oracle.py, oracle/multi_prompt_oracle.py and oracle/double_take_oracle.py:

  * dec_denoiser: multi-prompt guidance over K (tokens, mask) prompts (multi_prompt_oracle.compose);
  * transition_y: the conditioning of refined transitions, (tokens, mask) text_embed gathered per transition."""
import torch

from oracle import double_take_oracle as dt
from oracle import mdm_oracle as mo
from oracle import multi_prompt_oracle as mpo


def dec_denoiser(W, timestep_map, prompts, weight, lengths=None, mask_frames=True, cast=None):
    """denoise(x, i) of multi-prompt guidance on the BERT decoder: prompts a list of K (tokens [Mt_k, B, 768], padding
    mask [B, Mt_k]) pairs, each at its own Mt_k.  The unconditional prediction (mask_cond zeroes the tokens) admits every
    token some prompt admits, the prompts right-padded to the longest."""
    K = int(weight.shape[1])
    Mt = max(int(e.shape[0]) for e, _ in prompts[:K])
    B = int(prompts[0][1].shape[0])
    pad_u = torch.ones(B, Mt, dtype=torch.bool)
    for _, m in prompts[:K]:
        pad_u[:, :m.shape[1]] &= m.bool()
    enc_u = torch.zeros(Mt, B, prompts[0][0].shape[-1])

    def f(x, i):
        tm = int(timestep_map[i])
        prefix = x.new_zeros(x.shape[:-1] + (0,))
        xk = [mo.denoise_dec(W, x, tm, e, m, prefix, lengths, mask_frames, False, cast) for e, m in prompts[:K]]
        xu = mo.denoise_dec(W, x, tm, enc_u, pad_u, prefix, lengths, mask_frames, True, cast)
        return mpo.compose(xu, xk, weight)
    return f


def transition_y(y, lengths, motion_start, h, m, x_init):
    """double_take_oracle.transition_y for a y whose text_embed is a (tokens [Mt, B, C], mask [B, Mt]) pair: each
    transition takes its later window's token columns and mask rows (a single prompt [Mt, 1, C] / [1, Mt] stays
    shared)."""
    tok, msk = y["text_embed"]
    out = dt.transition_y(dict(y, text_embed=tok), lengths, motion_start, h, m, x_init)   # tokens: along dim 1
    bs = [b for _, b, _, _ in dt.layout(lengths, motion_start, h, m)]
    out["text_embed"] = (out["text_embed"], msk if msk.shape[0] == 1 else msk[bs])
    return out
