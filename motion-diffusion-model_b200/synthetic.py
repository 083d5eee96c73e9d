"""Deterministic synthetic checkpoints and inputs (no network => no released checkpoints).

`synthetic_state_dict` produces a reference-format ``state_dict`` (same key names and shapes as a
checkpoint written by the reference's train loop, SURVEY.md appendix A.4) from a numpy
``default_rng`` stream, so the very same weights can be regenerated in the build container, on the
GPU box and inside the reference oracle without shipping 70 MB files.  Scales follow the default
torch initialisers (Linear: U(+-1/sqrt(fan_in)); MHA in_proj: xavier-uniform) but biases and the
LayerNorm affine parameters are made non-trivial so that parity tests exercise them.
"""
import math

import numpy as np
import torch


def _uniform(rng, shape, bound):
    return torch.from_numpy(rng.uniform(-bound, bound, size=shape).astype(np.float32))


def _normal(rng, shape, std):
    return torch.from_numpy((rng.standard_normal(size=shape) * std).astype(np.float32))


HML_TARGET_JOINTS = ["pelvis", "left_foot", "right_foot", "left_wrist", "right_wrist", "head", "traj", "heading"]


def synthetic_state_dict(arch="trans_enc", latent_dim=512, ff_size=1024, num_layers=8, input_feats=263,
                         cond_dim=512, cond_mode="text", num_actions=1, seed=0, target_encoder=None, target_enc_layers=1,
                         target_joints=HML_TARGET_JOINTS, qk_gain=1.0, cross_qk_gain=1.0, ffn_gain=1.0, ln_outliers=0.0):
    """target_encoder ('single' / 'multi' / 'split', args.multi_encoder_type) adds the embed_target_cond.* tensors of
    that encoder (model/mdm.py:399-480) for the extended joint list `target_joints`, drawn from a stream of their own:
    every other tensor is the same as without them.

    Stress options for precision tests, applied after every draw (at their defaults the output is the init-scale
    checkpoint above, bit for bit).  They are stress settings chosen for testing, not statistics measured on a released
    checkpoint (none is available here); oracle/weight_families.py picks them from the statistic each one targets.
      qk_gain: the q and k rows of every self-attention in_proj (weight and bias) are scaled by it, so every
        self-attention logit is scaled by qk_gain**2 (sharper attention);
      cross_qk_gain: the same for the cross-attention of trans_dec;
      ffn_gain: linear1 (weight and bias) of every layer is scaled by it, and so is every FFN pre-activation;
      ln_outliers: this fraction of the channels of every LayerNorm get a bias of +-U(5, 10) (own stream)."""
    rng = np.random.default_rng(seed)
    d = latent_dim
    sd = {}

    def linear(prefix, out_f, in_f):
        b = 1.0 / math.sqrt(in_f)
        sd[prefix + ".weight"] = _uniform(rng, (out_f, in_f), b)
        sd[prefix + ".bias"] = _uniform(rng, (out_f,), b)

    def layer_norm(prefix):
        sd[prefix + ".weight"] = 1.0 + _normal(rng, (d,), 0.1)
        sd[prefix + ".bias"] = _normal(rng, (d,), 0.1)

    def mha(prefix):
        xb = math.sqrt(6.0 / (d + 3 * d))
        sd[prefix + ".in_proj_weight"] = _uniform(rng, (3 * d, d), xb)
        sd[prefix + ".in_proj_bias"] = _normal(rng, (3 * d,), 0.02)
        linear(prefix + ".out_proj", d, d)

    linear("input_process.poseEmbedding", d, input_feats)
    linear("embed_timestep.time_embed.0", d, d)
    linear("embed_timestep.time_embed.2", d, d)
    if "text" in cond_mode:
        linear("embed_text", d, cond_dim)
    if "action" in cond_mode:
        sd["embed_action.action_embedding"] = _normal(rng, (num_actions, d), 1.0)
    if arch == "trans_enc":
        for l in range(num_layers):
            p = "seqTransEncoder.layers.%d" % l
            mha(p + ".self_attn")
            linear(p + ".linear1", ff_size, d)
            linear(p + ".linear2", d, ff_size)
            layer_norm(p + ".norm1")
            layer_norm(p + ".norm2")
    elif arch == "trans_dec":
        for l in range(num_layers):
            p = "seqTransDecoder.layers.%d" % l
            mha(p + ".self_attn")
            mha(p + ".multihead_attn")
            linear(p + ".linear1", ff_size, d)
            linear(p + ".linear2", d, ff_size)
            layer_norm(p + ".norm1")
            layer_norm(p + ".norm2")
            layer_norm(p + ".norm3")
    else:
        raise ValueError("unsupported arch %r" % (arch,))
    linear("output_process.poseFinal", input_feats, d)
    if target_encoder is not None:
        rng = np.random.default_rng([seed, 0x7a5])
        n = len(target_joints)

        def mlp(prefix, d_in, width, n_hidden):
            linear(prefix + ".0", width, d_in)
            for k in range(1, n_hidden + 1):
                linear(prefix + ".%d" % (2 * k), width, width)
        if target_encoder == "single":
            mlp("embed_target_cond.mlp", 4 * n, d, target_enc_layers)
        elif target_encoder == "split":
            for i in range(n):
                mlp("embed_target_cond.mini_mlps.%d" % i, 4, d // n, target_enc_layers)
        elif target_encoder == "multi":
            for j in target_joints:
                mlp("embed_target_cond.target_loc_emb." + j, 3, d, 1)
            # WeightedSum weights (randn init): kept away from a zero sum so that w / w.sum() stays moderate
            sd["embed_target_cond.target_all_loc_emb.weights"] = torch.from_numpy(
                rng.uniform(0.25, 1.0, size=n).astype(np.float32) * np.where(np.arange(n) % 3 == 2, -0.5, 1.0).astype(np.float32))
        else:
            raise ValueError("unsupported target encoder %r" % (target_encoder,))
    _stress(sd, seed, d, qk_gain, cross_qk_gain, ffn_gain, ln_outliers)
    return sd


def _stress(sd, seed, d, qk_gain, cross_qk_gain, ffn_gain, ln_outliers):
    """The stress options of synthetic_state_dict, in place."""
    for name, t in list(sd.items()):
        if ".linear1." in name and ffn_gain != 1.0:
            sd[name] = t * ffn_gain
        for key, gain in ((".self_attn.in_proj_", qk_gain), (".multihead_attn.in_proj_", cross_qk_gain)):
            if key in name and gain != 1.0:
                t = t.clone()
                t[: 2 * d] *= gain                # q and k rows; v keeps its scale
                sd[name] = t
    if ln_outliers > 0.0:
        rng = np.random.default_rng([seed, 0x1b5])
        n = max(1, int(round(ln_outliers * d)))
        for name in sorted(k for k in sd if ".norm" in k and k.endswith(".bias")):
            ch = rng.choice(d, size=n, replace=False)
            t = sd[name].clone()
            t[ch] = torch.from_numpy((rng.uniform(5.0, 10.0, size=n) * rng.choice([-1.0, 1.0], size=n)).astype(np.float32))
            sd[name] = t


def synthetic_target_inputs(batch, joint_names=HML_TARGET_JOINTS, seed=5):
    """Deterministic target-location conditioning in the reference's y schema (model/mdm.py:197-199):
    target_cond [B, n_ext, 3] fp32 (every joint has values, valid or not), target_joint_names (per sample, a numpy array
    of names: the layout CLoSD passes), is_heading [B] bool.  The joint sets cycle through mixed choices, some with
    heading; the last sample (of a batch of 3 or more) has no joint and no heading."""
    rng = np.random.default_rng(seed)
    target = torch.from_numpy(rng.standard_normal(size=(batch, len(joint_names), 3)).astype(np.float32))
    goal = [j for j in joint_names if j not in ("heading",)]
    choices = [["pelvis", "head"], ["traj"], ["left_wrist", "right_wrist", "left_foot"], goal, ["right_foot"]]
    names, heading = [], []
    for b in range(batch):
        if batch >= 3 and b == batch - 1:
            names.append(np.array([], dtype="<U16"))
            heading.append(False)
            continue
        names.append(np.array([j for j in choices[b % len(choices)] if j in joint_names]))
        heading.append(b % 2 == 0)
    return dict(target_cond=target, target_joint_names=names, is_heading=torch.tensor(heading))


def synthetic_inputs(batch, njoints=263, nfeats=1, nframes=196, steps=50, cond_dim=512, seed=10,
                     lengths=None, scale=2.5, dtype=torch.float32):
    """Noise tape [x_T, eps_{T-1} .. eps_0], text embedding [1,B,cond_dim], lengths, mask, scale."""
    rng = np.random.default_rng(seed)
    shape = (batch, njoints, nfeats, nframes)
    tape = [torch.from_numpy(rng.standard_normal(size=shape).astype(np.float32)) for _ in range(steps + 1)]
    text_embed = torch.from_numpy(rng.standard_normal(size=(1, batch, cond_dim)).astype(np.float32))
    if lengths is None:
        lengths = [nframes] * batch
    lengths = torch.tensor(lengths, dtype=torch.int64)
    mask = (torch.arange(nframes)[None, :] < lengths[:, None]).view(batch, 1, 1, nframes)
    if not torch.is_tensor(scale):
        scale = torch.full((batch,), float(scale), dtype=torch.float32)
    return dict(tape=tape, text_embed=text_embed, lengths=lengths, mask=mask, scale=scale)


def synthetic_dip_inputs(batch, n_tokens, context_len, njoints=263, nfeats=1, cond_dim=768, seed=3):
    """Deterministic DiP conditioning in the reference's layouts (model/mdm.py:180-187,204): BERT token features
    [n_tokens, B, 768], ragged padding mask [B, n_tokens] (True = padding; sample 0 has none), prefix [B, J, F, ctx]."""
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(n_tokens, batch, cond_dim, generator=g)
    tmask = torch.zeros(batch, n_tokens, dtype=torch.bool)
    for b in range(1, batch):
        tmask[b, n_tokens - (b * 2) % n_tokens:] = True
    prefix = torch.randn(batch, njoints, nfeats, context_len, generator=g)
    return enc, tmask, prefix


def synthetic_norm_stats(dim=263, seed=7):
    """Stand-in for the dataset's Mean.npy / Std.npy (data_loaders/humanml/data/dataset.py:248-249): fp32 [dim]."""
    rng = np.random.default_rng(seed)
    mean = rng.standard_normal(dim).astype(np.float32)
    std = rng.uniform(0.2, 2.0, size=dim).astype(np.float32)
    return torch.from_numpy(mean), torch.from_numpy(std)
