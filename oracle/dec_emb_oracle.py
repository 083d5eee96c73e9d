"""TEST INFRASTRUCTURE ONLY -- plain-torch fp32 restatement of MDM.forward for arch='trans_dec' with
text_encoder_type='clip' and emb_trans_dec=True (the humanml-decoder-with-emb checkpoint), on top of the layer
restatements of oracle/mdm_oracle.py.  Pinned against the live reference by tests/golden/dec_emb_*.npz
(oracle/gen_golden_dec_emb.py) and tests/test_dec_emb_cpu.py.

Reference lines (model/mdm.py): time_emb (+ the target term, :197-199); text_emb = embed_text(mask_cond(clip)) (:218);
memory = text_emb + time_emb, ONE token per sample, no memory mask (:220, :262-263); tgt = cat(time_emb, frames) + pe
(:256-258); tgt_key_padding_mask = ~mask with a False column for token 0 when mask_frames (:241-247); output [1:]
(:269-270).  The decoder layers are nn.TransformerDecoderLayer, post-norm (mdm_oracle.decoder_stack).

`cast` rounds every GEMM operand through a narrower dtype, as in mdm_oracle; it exists for the precision study of
DESIGN.md section 2 and is None for parity work.  `cast=mo.DEC_EMB_SITES` is the site-exact fp16 emulation of the
engine (mdm_oracle.Sites).
"""
import torch

from . import mdm_oracle as mo


def denoise_dec_emb(W, x, t_model, cond, lengths=None, mask_frames=True, uncond=False, g=None, cast=None):
    """x [B,J,F,T]; t_model python int; cond = text_embed [1,B,512] (or [1,1,512]); g [B,d] target embedding or None;
    lengths [B] valid frames or None (=> no key mask)."""
    B, J, Fe, T = x.shape
    h, mem, keymask = dec_emb_input(W, x, t_model, cond, lengths, mask_frames, uncond, g, cast)
    h = mo.decoder_stack(W, h, mem, keymask, None, cast)[:, 1:]
    out = mo._lin(h, W["output_process.poseFinal.weight"], W["output_process.poseFinal.bias"], cast)
    return out.reshape(B, T, J, Fe).permute(0, 2, 3, 1).contiguous()


def dec_emb_input(W, x, t_model, cond, lengths=None, mask_frames=True, uncond=False, g=None, cast=None):
    """The decoder stack's inputs of denoise_dec_emb: (h [B, T+1, d], memory [B, 1, d], key mask or None)."""
    B, J, Fe, T = x.shape
    d = W.d
    temb = mo.timestep_embedding(W, t_model)[None, :].expand(B, d)
    if g is not None:
        temb = temb + g
    c = cond[0].expand(B, -1)
    if uncond:                                                              # mask_cond force_mask
        c = torch.zeros_like(c)
    mem = (mo._lin(c, W["embed_text.weight"], W["embed_text.bias"], None) + temb)[:, None, :]   # [B, 1, d]
    frames = x.permute(0, 3, 1, 2).reshape(B, T, J * Fe)
    hf = mo._lin(frames, W["input_process.poseEmbedding.weight"], W["input_process.poseEmbedding.bias"], cast)
    h = torch.cat([temb[:, None, :], hf], dim=1) + W.pe[: T + 1][None]
    keymask = None
    if mask_frames and lengths is not None and T > 1:
        keymask = torch.arange(T + 1)[None, :] >= (lengths[:, None] + 1)
    return h, mem, keymask


def cfg_denoise_dec_emb(W, x, t_model, cond, scale, lengths=None, mask_frames=True, g=None, cast=None):
    """ClassifierFreeSampleModel.forward (utils/sampler_util.py:27-34): both halves keep the target term."""
    oc = denoise_dec_emb(W, x, t_model, cond, lengths, mask_frames, False, g, cast)
    ou = denoise_dec_emb(W, x, t_model, cond, lengths, mask_frames, True, g, cast)
    return ou + scale.view(-1, 1, 1, 1) * (oc - ou)


def denoiser(W, timestep_map, cond, scale, lengths=None, mask_frames=True, g=None, cast=None):
    """denoise(x, i) at schedule index i (the model timestep is timestep_map[i]; i = -1 wraps, as PLMS needs),
    CFG-wrapped when `scale` is given -- the interface of plms_oracle.plms_loop and reverse_oracle.reverse_loop."""
    def f(x, i):
        tm = int(timestep_map[i])
        if scale is None:
            return denoise_dec_emb(W, x, tm, cond, lengths, mask_frames, False, g, cast)
        return cfg_denoise_dec_emb(W, x, tm, cond, scale, lengths, mask_frames, g, cast)
    return f


def sample_loop(denoise, tables, tape, sampler="ddpm", eta=0.0, inpaint=None, collect=None):
    """p_sample_loop / ddim_sample_loop with the noise tape [x_T, eps_{n-1}, ..., eps_0] (mdm_oracle.sample_loop's
    update rules, any denoiser); `collect` receives every step's sample."""
    n = len(tables["betas"])
    x = tape[0].clone()
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = denoise(x, i)
        eps = tape[1 + k]
        if sampler == "ddpm":
            x, _ = mo.p_sample_step(tables, x0, x, i, eps, inpaint)
        else:
            if inpaint is not None:
                m, motion = inpaint
                x0 = (x0 * ~m) + (motion * m)
            x = mo.ddim_step(tables, x0, x, i, eps, eta)
        if collect is not None:
            collect.append(x.clone())
    return x
