"""TEST INFRASTRUCTURE ONLY -- weight families for the precision tests: synthetic checkpoints whose layer-0 statistics,
measured with the fp32 oracle on a probe input, reach a chosen target.

  init          synthetic_state_dict as it is (default torch initialisers)
  sharp_attn8   the q and k rows of every self-attention (and of the DiP cross-attention) scaled so that the median
  sharp_attn16  per-row spread of layer 0's logits (max - median over the valid keys, valid query rows) is 8 / 16
  wide_ffn      linear1 scaled so that 1% of layer 0's FFN pre-activations (valid tokens) exceed 6 in magnitude
  ln_shift      1% of the channels of every LayerNorm get a bias of +-U(5, 10)

These are stress settings chosen for testing, not statistics measured on a released checkpoint (none is available
here).  A trained model's attention is sharper and its activations larger than at init scale, and the engine stores
q / k / v, P, the attention output and the GELU output in fp16, whose error grows with those magnitudes.
"""
import math

import torch
import torch.nn.functional as F

from . import dec_emb_oracle as deo
from . import mdm_oracle as mo

FAMILIES = ("init", "sharp_attn8", "sharp_attn16", "wide_ffn", "ln_shift")
FFN_LIMIT, FFN_FRACTION = 6.0, 0.01
LN_OUTLIERS, LN_OUTLIER_MIN = 0.01, 5.0


def _spread(hq, hk, in_w, in_b, H, qvalid, kvalid):
    """Median over (sample, head, valid query) of max - median of the logits over the valid keys."""
    B, Sq, d = hq.shape
    dh = d // H
    q = (hq @ in_w[:d].t() + in_b[:d]).view(B, Sq, H, dh).transpose(1, 2)
    k = (hk @ in_w[d:2 * d].t() + in_b[d:2 * d]).view(B, hk.shape[1], H, dh).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
    rows = []
    for b in range(B):
        sb = s[b][:, qvalid[b]][:, :, kvalid[b]]
        rows.append((sb.amax(-1) - sb.median(-1).values).flatten())
    return torch.cat(rows).median().item()


def _mha(W, p):
    return dict(in_w=W[p + "in_proj_weight"], in_b=W[p + "in_proj_bias"], out_w=W[p + "out_proj.weight"],
                out_b=W[p + "out_proj.bias"])


def layer0_stats(W, h, keymask=None, mem=None, memmask=None):
    """Layer 0 of the fp32 oracle on its input h [B, S, d] (mem: the decoder's memory): the self-attention logit
    spread, the cross-attention logit spread (memories of more than one token), and the 99th percentile and the
    fraction above FFN_LIMIT of |FFN pre-activation| over the valid tokens."""
    p = ("seqTransDecoder" if mem is not None else "seqTransEncoder") + ".layers.0."
    B, S, d = h.shape
    valid = ~keymask if keymask is not None else torch.ones(B, S, dtype=torch.bool)
    st = dict(self_spread=_spread(h, h, W[p + "self_attn.in_proj_weight"], W[p + "self_attn.in_proj_bias"], W.H,
                                  valid, valid))
    h = F.layer_norm(h + mo._mha_self(h, _mha(W, p + "self_attn."), keymask, W.H), (d,), W[p + "norm1.weight"],
                     W[p + "norm1.bias"], 1e-5)
    if mem is not None:
        ca = _mha(W, p + "multihead_attn.")
        if mem.shape[1] > 1:
            mvalid = ~memmask if memmask is not None else torch.ones(B, mem.shape[1], dtype=torch.bool)
            st["cross_spread"] = _spread(h, mem, ca["in_w"], ca["in_b"], W.H, valid, mvalid)
        h = F.layer_norm(h + mo._mha_cross(h, mem, ca, memmask, W.H), (d,), W[p + "norm2.weight"], W[p + "norm2.bias"],
                         1e-5)
    pre = (h @ W[p + "linear1.weight"].t() + W[p + "linear1.bias"])[valid].abs().flatten()
    st["ffn_q99"] = torch.quantile(pre.double(), 1.0 - FFN_FRACTION).item()
    st["ffn_frac"] = (pre > FFN_LIMIT).double().mean().item()
    return st


def ln_outlier_fraction(sd):
    """Fraction of all LayerNorm bias channels with |beta| >= LN_OUTLIER_MIN."""
    b = torch.cat([v.flatten() for k, v in sd.items() if ".norm" in k and k.endswith(".bias")])
    return (b.abs() >= LN_OUTLIER_MIN).double().mean().item()


def family_state_dict(family, make_sd, probe):
    """(state_dict, statistics) of `family`.  make_sd(**stress options) -> synthetic_state_dict with those options
    (qk_gain, cross_qk_gain, ffn_gain, ln_outliers); probe(W) -> dict(h=, keymask=, mem=, memmask=), layer 0's input
    for the oracle weights W (enc_probe / dip_probe / dec_emb_probe).  The statistics are those of the returned
    weights, with the options that produced them."""
    def stats(sd):
        W = mo.OracleWeights(sd, 1)
        with torch.no_grad():
            st = layer0_stats(W, **probe(W))
        st["ln_outlier_frac"] = ln_outlier_fraction(sd)
        return st

    opts = {}
    if family.startswith("sharp_attn"):
        target = float(family[len("sharp_attn"):])
        opts["qk_gain"] = math.sqrt(target / stats(make_sd())["self_spread"])      # logits scale with the gain squared
        st = stats(make_sd(**opts))
        if "cross_spread" in st:
            opts["cross_qk_gain"] = math.sqrt(target / st["cross_spread"])
    elif family == "wide_ffn":
        opts["ffn_gain"] = FFN_LIMIT / stats(make_sd())["ffn_q99"]                # pre-activations scale with the gain
    elif family == "ln_shift":
        opts["ln_outliers"] = LN_OUTLIERS
    elif family != "init":
        raise ValueError("unknown weight family %r (known: %s)" % (family, ", ".join(FAMILIES)))
    sd = make_sd(**opts)
    st = stats(sd)
    st.update(opts)
    return sd, st


def enc_probe(x, t_model, cond, lengths=None, action=None):
    """Layer 0's input of denoise_enc (conditional half)."""
    def probe(W):
        h, keymask = mo.enc_input(W, x, t_model, cond, lengths, action=action)
        return dict(h=h, keymask=keymask)
    return probe


def dip_probe(x, t_model, enc_text, text_mask, prefix, lengths=None):
    """Layer 0's input of denoise_dec (conditional half)."""
    def probe(W):
        h, mem, keymask = mo.dec_input(W, x, t_model, enc_text, prefix, lengths)
        return dict(h=h, keymask=keymask, mem=mem, memmask=text_mask)
    return probe


def dec_emb_probe(x, t_model, cond, lengths=None):
    """Layer 0's input of denoise_dec_emb (conditional half)."""
    def probe(W):
        h, mem, keymask = deo.dec_emb_input(W, x, t_model, cond, lengths)
        return dict(h=h, keymask=keymask, mem=mem)
    return probe
