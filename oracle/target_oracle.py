"""TEST INFRASTRUCTURE ONLY -- plain-torch fp32 restatement of target-location conditioning (multi_target_cond), on
top of oracle/mdm_oracle.py.  The product path never imports it.

What is restated (paths relative to the reference repository root):
  * EmbedTargetLocSingle / Split / Multi ...... model/mdm.py:399-480
  * WeightedSum ................................ utils/misc.py:5-16
  * the target term of MDM.forward ............. model/mdm.py:197-199: time_emb += embed_target_cond(...), in both
                                                 halves of a CFG pair (utils/sampler_util.py:27-34 never sets
                                                 target_uncond)
Pinned by tests/golden/{dip,enc}_target_small.npz, which oracle/gen_golden_target.py makes from the reference itself.
"""
import torch
import torch.nn.functional as F

from . import mdm_oracle as mo


def validity(joint_names, target_joint_names, is_heading):
    """[B, n_ext] fp32: 1 for each named joint, plus 'heading' when is_heading[b] (model/mdm.py:410-416)."""
    v = torch.zeros(len(target_joint_names), len(joint_names))
    for b, names in enumerate(target_joint_names):
        for j in list(names) + (["heading"] if bool(is_heading[b]) else []):
            v[b, joint_names.index(str(j))] = 1.0
    return v


def target_embedding(W, encoder, target, valid, layers=1, joint_names=None):
    """g [B, d] = embed_target_cond(target [B, n, 3], validity [B, n]) for encoder 'single', 'split' or 'multi'
    (joint_names: the extended joint list, which names the multi encoder's per-joint MLPs)."""
    B, n, _ = target.shape
    x = torch.cat([target, valid[..., None]], dim=-1)                       # [B, n, 4]

    def mlp(prefix, h, n_hidden):
        h = mo._lin(h, W[prefix + "0.weight"], W[prefix + "0.bias"])
        for k in range(1, n_hidden + 1):
            h = mo._lin(F.silu(h), W[prefix + "%d.weight" % (2 * k)], W[prefix + "%d.bias" % (2 * k)])
        return h
    if encoder == "single":
        return mlp("embed_target_cond.mlp.", x.reshape(B, 4 * n), layers)
    if encoder == "split":
        return torch.cat([mlp("embed_target_cond.mini_mlps.%d." % i, x[:, i], layers) for i in range(n)], dim=-1)
    if encoder == "multi":
        names = joint_names
        w = W["embed_target_cond.target_all_loc_emb.weights"]
        out = torch.zeros(B, W.d)
        for b in range(B):
            rows = torch.zeros(n, W.d)
            for i in range(n):
                if valid[b, i] > 0:
                    rows[i] = mlp("embed_target_cond.target_loc_emb.%s." % names[i], target[b, i], 1)
            out[b] = (w / w.sum()) @ rows
        return out
    raise ValueError(encoder)


def denoise_enc(W, x, t_model, cond, g, lengths=None, mask_frames=True, uncond=False):
    """MDM.forward, trans_enc, text or no_cond, with the target term: token 0 = text_emb + (temb + g)."""
    B, J, Fe, T = x.shape
    temb = mo.timestep_embedding(W, t_model)[None, :].expand(B, W.d)
    if g is not None:
        temb = temb + g
    if cond is not None:
        c = torch.zeros_like(cond[0]) if uncond else cond[0]
        tok0 = mo._lin(c, W["embed_text.weight"], W["embed_text.bias"]) + temb
    else:
        tok0 = temb
    frames = x.permute(0, 3, 1, 2).reshape(B, T, J * Fe)
    hf = mo._lin(frames, W["input_process.poseEmbedding.weight"], W["input_process.poseEmbedding.bias"])
    h = torch.cat([tok0[:, None, :], hf], dim=1) + W.pe[: T + 1][None]
    keymask = None
    if mask_frames and lengths is not None and T > 1:
        keymask = torch.arange(T + 1)[None, :] >= (lengths[:, None] + 1)
    h = mo.encoder_stack(W, h, keymask)[:, 1:]
    out = mo._lin(h, W["output_process.poseFinal.weight"], W["output_process.poseFinal.bias"])
    return out.reshape(B, T, J, Fe).permute(0, 2, 3, 1).contiguous()


def denoise_dec(W, x, t_model, enc_text, text_mask, prefix, g, lengths=None, mask_frames=True, uncond=False):
    """MDM.forward, DiP, with the target term: memory token m = text_emb[m] + (temb + g)."""
    B, J, Fe, Tp = x.shape
    ctx = prefix.shape[-1]
    temb = mo.timestep_embedding(W, t_model)[None, :].expand(B, W.d)
    if g is not None:
        temb = temb + g
    enc = torch.zeros_like(enc_text) if uncond else enc_text
    mem = mo._lin(enc.permute(1, 0, 2), W["embed_text.weight"], W["embed_text.bias"]) + temb[:, None, :]
    xf = torch.cat([prefix, x], dim=-1)
    T = ctx + Tp
    frames = xf.permute(0, 3, 1, 2).reshape(B, T, J * Fe)
    h = mo._lin(frames, W["input_process.poseEmbedding.weight"], W["input_process.poseEmbedding.bias"]) + W.pe[:T][None]
    keymask = None
    if mask_frames and lengths is not None and T > 1:
        keymask = torch.arange(T)[None, :] >= (lengths[:, None] + ctx)
    h = mo.decoder_stack(W, h, mem, keymask, text_mask)[:, ctx:]
    out = mo._lin(h, W["output_process.poseFinal.weight"], W["output_process.poseFinal.bias"])
    return out.reshape(B, Tp, J, Fe).permute(0, 2, 3, 1).contiguous()


def cfg(fn, scale, *args, **kw):
    """ClassifierFreeSampleModel.forward: both halves keep g."""
    oc = fn(*args, uncond=False, **kw)
    ou = fn(*args, uncond=True, **kw)
    return ou + scale.view(-1, 1, 1, 1) * (oc - ou)


def sample_loop_enc(W, tables, timestep_map, tape, cond, g, scale, lengths=None, mask_frames=True):
    n = len(tables["betas"])
    x = tape[0].clone()
    for k, i in enumerate(range(n - 1, -1, -1)):
        tm = int(timestep_map[i])
        x0 = cfg(denoise_enc, scale, W, x, tm, cond, g, lengths, mask_frames)
        x, _ = mo.p_sample_step(tables, x0, x, i, tape[1 + k])
    return x


def sample_loop_dec(W, tables, timestep_map, tape, enc_text, text_mask, prefix, g, scale, lengths=None,
                    mask_frames=True):
    n = len(tables["betas"])
    x = tape[0].clone()
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = cfg(denoise_dec, scale, W, x, int(timestep_map[i]), enc_text, text_mask, prefix, g, lengths, mask_frames)
        x, _ = mo.p_sample_step(tables, x0, x, i, tape[1 + k])
    return x
