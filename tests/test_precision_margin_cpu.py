"""CPU: the pieces behind tests/test_precision_margin_gpu.py -- the weight families reach their target statistics
deterministically, the stress options leave the default synthetic checkpoint unchanged, and the site-exact fp16
emulation (mdm_oracle.Sites) is the plain oracle without sites and moves the output at every site it names."""
import hashlib
import importlib

import pytest
import torch

from oracle import mdm_oracle as mo, weight_families as wf
from precision_cases import KINDS, T_HI

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")


def _sha(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].numpy().tobytes())
    return h.hexdigest()


def test_default_state_dict_unchanged():
    """The weights every other test and the benchmark use, bit for bit (hashes of the checkpoints before the stress
    options existed); explicit default options change nothing either."""
    enc = syn.synthetic_state_dict(num_layers=2, seed=3)
    dec = syn.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=3)
    assert _sha(enc) == "535d72098a4c24ec2bee2829c66fb83211f98443c1f3b03c16768404e0dfedff"
    assert _sha(dec) == "45f6c5ba7540be92a630a1a4407f64664e6a9b9982d5c70ad938bb1017f811ae"
    same = syn.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=3, qk_gain=1.0, cross_qk_gain=1.0,
                                    ffn_gain=1.0, ln_outliers=0.0)
    assert _sha(same) == _sha(dec)


def test_stress_options_touch_only_their_tensors():
    base = syn.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=3)
    d = 512
    for opts, hit in ((dict(qk_gain=2.0), ".self_attn.in_proj_"), (dict(cross_qk_gain=2.0), ".multihead_attn.in_proj_"),
                      (dict(ffn_gain=2.0), ".linear1."), (dict(ln_outliers=0.01), ".bias")):
        sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=3, **opts)
        for k, v in sd.items():
            if hit not in k or (hit == ".bias" and ".norm" not in k):
                assert torch.equal(v, base[k]), (opts, k)
            elif "in_proj" in hit:
                assert torch.equal(v[: 2 * d], base[k][: 2 * d] * 2.0) and torch.equal(v[2 * d:], base[k][2 * d:]), k
            elif hit == ".linear1.":
                assert torch.equal(v, base[k] * 2.0), k
            else:
                changed = v != base[k]
                assert changed.sum() == 5 and ((v[changed].abs() >= 5) & (v[changed].abs() <= 10)).all(), k


@pytest.mark.parametrize("kind", list(KINDS))
def test_families_reach_their_targets(kind):
    k = KINDS[kind]()
    for family in wf.FAMILIES:
        sd, st = wf.family_state_dict(family, k.make_sd, k.probe)
        sd2, st2 = wf.family_state_dict(family, k.make_sd, k.probe)
        assert st == st2 and all(torch.equal(sd[n], sd2[n]) for n in sd), family      # deterministic
        print("%s / %s: %s" % (kind, family, st))
        if family.startswith("sharp_attn"):
            target = float(family[len("sharp_attn"):])
            assert abs(st["self_spread"] / target - 1) < 1e-3, st
            if kind == "dip":
                assert abs(st["cross_spread"] / target - 1) < 1e-3, st
        elif family == "wide_ffn":
            assert 0.009 <= st["ffn_frac"] <= 0.011, st
        elif family == "ln_shift":
            assert 0.009 <= st["ln_outlier_frac"] <= 0.011, st
        else:
            assert st["self_spread"] < 2 and st["ffn_frac"] < 1e-3 and st["ln_outlier_frac"] == 0, st


def _forward(k, cast):
    W = mo.OracleWeights(k.make_sd(), 2)
    with torch.no_grad():
        return k.forward(W, k.inp["tape"][0], T_HI, cast)


@pytest.mark.parametrize("kind", list(KINDS))
def test_emulation_without_sites_is_the_oracle(kind):
    k = KINDS[kind]()
    assert torch.equal(_forward(k, mo.Sites()), _forward(k, None))


@pytest.mark.parametrize("kind", ["trans_enc_text", "dip", "dec_emb"])
def test_every_site_moves_the_output(kind):
    """Each site the model's emulation rounds changes the output alone; so do DiP's [hi | lo] sites (which its engine
    keeps unrounded) and the CLIP decoder's fp32 cross-attention must not see the cross-attention sites."""
    k = KINDS[kind]()
    plain = _forward(k, None)
    sites = set(k.sites) | ({"attn", "ffn_in", "gelu"} if kind == "dip" else set())
    for s in sorted(sites):
        assert not torch.equal(_forward(k, mo.Sites({s})), plain), s
    if kind == "dec_emb":
        cross = {"cross_q_in", "cross_q", "mem", "cross_kv", "cross_attn", "cross_weights"}
        assert not cross & k.sites
