"""CPU: multi-prompt guidance (MultiPromptSampleModel, b200mdm_set_cond_multi / _dec / b200mdm_set_prompt_weight;
DESIGN.md "Multi-prompt guidance").

  * the oracle's composition with K = 1 and w = scale is the oracle's classifier-free guidance within fp32 rounding, and
    its fp32 composition agrees with the fp64 one;
  * body_part_mask matches the reference's HML_LOWER_BODY_MASK / HML_UPPER_BODY_MASK (tests/golden/hml_body_masks.npz);
  * every refusal of the wrapper and the samplers that needs no GPU, and y is never mutated by them;
  * parallel.shard_model_kwargs slices the new keys; the C ABI's argument checks, which run before any CUDA call."""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import ROOT, default_args, rel_err
from oracle import mdm_oracle as mo
from oracle import multi_prompt_oracle as mpo

syn = b200mdm.synthetic


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_oracle_k1_is_cfg():
    L, B, T = 2, 3, 16
    sd = syn.synthetic_state_dict(num_layers=L, seed=3)
    inp = syn.synthetic_inputs(B, nframes=T, steps=0, seed=4, lengths=[16, 9, 2], scale=torch.tensor([2.5, 1.0, 7.5]))
    W = mo.OracleWeights(sd, L)
    x, te, sc, ln = inp["tape"][0], inp["text_embed"], inp["scale"], inp["lengths"]
    cfg = mo.cfg_denoise_enc(W, x, 7, te, sc, ln)
    f = mpo.enc_denoiser(W, list(range(10)), te, sc.view(B, 1, 1, 1), ln)
    got = f(x, 7)
    assert rel_err(got, cfg) < 1e-6
    oc = mo.denoise_enc(W, x, 7, te, ln)
    ou = mo.denoise_enc(W, x, 7, te, ln, uncond=True)
    want64 = mpo.compose(ou.double(), [oc.double()], sc.double().view(B, 1, 1, 1))
    assert rel_err(got, want64) < 1e-6


def test_oracle_compose_order_and_broadcast():
    g = torch.Generator().manual_seed(0)
    xu, xa, xb = (torch.randn(2, 263, 1, 5, generator=g) for _ in range(3))
    w = torch.randn(2, 2, 1, 5, generator=g)
    got = mpo.compose(xu, [xa, xb], w)
    u = xu.reshape(2, 263, 5)
    want = (u + w[:, 0] * (xa.reshape(2, 263, 5) - u)) + w[:, 1] * (xb.reshape(2, 263, 5) - u)
    assert torch.equal(got.reshape(2, 263, 5), want)


def test_body_part_mask_matches_reference_fixture(golden):
    g = golden("hml_body_masks.npz")
    lower, upper = b200mdm.body_part_mask("lower"), b200mdm.body_part_mask("upper")
    assert lower.dtype == torch.bool and lower.shape == (263,)
    assert np.array_equal(lower.numpy(), g["lower"]) and np.array_equal(upper.numpy(), g["upper"])
    assert bool(b200mdm.body_part_mask(["lower", "upper"]).all()) and not bool((lower & upper).any())
    for bad in ("arms", [], ["lower", "head"]):
        with pytest.raises(ValueError):
            b200mdm.body_part_mask(bad)


def test_wrapper_and_sampler_refusals():
    model, diffusion = _model()
    mp = b200mdm.MultiPromptSampleModel(model)
    assert mp.njoints == 263 and mp.cond_mask_prob == 0.1
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    for wrapped in (cfg, b200mdm.HandshakeSampleModel(cfg, 2), SimpleNamespace(model=model)):
        with pytest.raises(TypeError):
            b200mdm.MultiPromptSampleModel(wrapped)
    with pytest.raises(TypeError):
        b200mdm.HandshakeSampleModel(mp, 2)
    with pytest.raises(TypeError):
        b200mdm.JointControlSampleModel(mp, torch.zeros(263), torch.ones(263), 1e-3, 4)
    dip, _ = _model(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    with pytest.raises(NotImplementedError):
        b200mdm.MultiPromptSampleModel(dip)
    uncond, _ = _model(unconstrained=True, cond_mask_prob=0.0)
    with pytest.raises(AssertionError):
        b200mdm.MultiPromptSampleModel(uncond)
    B, K, T = 2, 2, 24
    x = torch.zeros(B, 263, 1, T)
    t = torch.zeros(B, dtype=torch.long)
    y = {"prompt_embed": torch.zeros(K, B, 512), "prompt_weight": torch.ones(B, K, 1, 1), "lengths": torch.tensor([24, 7])}
    with pytest.raises(NotImplementedError):
        diffusion.calc_bpd_loop(mp, x, model_kwargs={"y": y})
    with pytest.raises(TypeError):
        b200mdm.refine_transitions(diffusion.p_sample_loop, mp, x, {"y": y}, 2, 2, 1)
    # y: missing or mis-shaped keys, non-finite weights, K out of range; raised before any engine work, y untouched
    snapshot = dict(y)
    for bad in ({"prompt_weight": None}, {"prompt_embed": None}, {"prompt_weight": torch.ones(B, K, 262, 1)},
                {"prompt_weight": torch.ones(B, K, 1, T + 1)}, {"prompt_weight": torch.ones(B + 1, K, 1, 1)},
                {"prompt_weight": torch.ones(B, K, 1)}, {"prompt_weight": torch.ones(B, K, 1, 1, dtype=torch.long)},
                {"prompt_weight": torch.full((B, K, 1, 1), float("nan"))},
                {"prompt_weight": torch.full((B, K, 1, 1), float("inf"))},
                {"prompt_weight": torch.ones(B, 0, 1, 1), "prompt_embed": torch.zeros(0, B, 512)},
                {"prompt_weight": torch.ones(B, 9, 1, 1), "prompt_embed": torch.zeros(9, B, 512)},
                {"prompt_embed": torch.zeros(K + 1, B, 512)}, {"prompt_embed": torch.zeros(K, B, 511)},
                {"prompt_embed": None, "prompt_text": [["a", "b"], ["c"]]},
                {"prompt_embed": None, "prompt_text": ["ab", "cd"]}):
        yy = {k: v for k, v in dict(y, **bad).items() if v is not None}
        for call in (lambda: diffusion.p_sample_loop(mp, x.shape, model_kwargs={"y": yy}),
                     lambda: diffusion.ddim_sample(mp, x, t, model_kwargs={"y": yy}),
                     lambda: mp(x, t, y=yy)):
            with pytest.raises(ValueError):
                call()
        assert "prompt_embed" not in yy or "prompt_embed" in bad or yy["prompt_embed"] is y["prompt_embed"]
    assert y.keys() == snapshot.keys() and all(y[k] is snapshot[k] for k in y)
    a2m, _ = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, dataset="humanact12"),
                                                SimpleNamespace(dataset=SimpleNamespace(num_actions=12)))
    ma = b200mdm.MultiPromptSampleModel(a2m)
    xa = torch.zeros(B, a2m.njoints, a2m.nfeats, T)
    w = torch.ones(B, K, 1, 1)
    for bad in (None, torch.zeros(B, K + 1, dtype=torch.long), torch.zeros(B, K), torch.full((B, K), 12),
                torch.full((B, K), -1)):
        ya = {"prompt_weight": w} if bad is None else {"prompt_weight": w, "prompt_action": bad}
        with pytest.raises(ValueError):
            ma.prompts(ya, xa.shape)
    e, a, ww = ma.prompts({"prompt_weight": w, "prompt_action": torch.tensor([[1, 2], [3, 11]])}, xa.shape)
    assert e is None and a.dtype == np.int64 and a.tolist() == [[1, 2], [3, 11]] and ww.dtype == torch.float32


def test_shard_model_kwargs_slices_the_prompt_keys():
    y = {"prompt_embed": torch.randn(2, 6, 512), "prompt_weight": torch.rand(6, 2, 263, 4),
         "prompt_action": torch.arange(12).view(6, 2), "prompt_text": [["a%d" % b, "b%d" % b] for b in range(6)]}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(part["prompt_embed"], y["prompt_embed"][:, 2:5])
    assert torch.equal(part["prompt_weight"], y["prompt_weight"][2:5])
    assert torch.equal(part["prompt_action"], y["prompt_action"][2:5])
    assert part["prompt_text"] == y["prompt_text"][2:5]


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    assert lib.b200mdm_set_cond_multi(None, 2, 24, 2, buf, None, None, None) == _lib.EINVAL
    assert lib.b200mdm_set_cond_multi_dec(None, 2, 24, 2, buf, None, None) == _lib.EINVAL
    assert lib.b200mdm_set_prompt_weight(None, 2, buf, 0, 0, 0, 0, None) == _lib.EINVAL
    assert b"null" in lib.b200mdm_last_error()


def test_symbols_in_header_and_lib():
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    assert "#define B200MDM_MAX_PROMPTS %d" % _lib.MAX_PROMPTS in header
    for name in ("b200mdm_set_cond_multi", "b200mdm_set_cond_multi_dec", "b200mdm_set_prompt_weight"):
        assert name + "(" in header and name in _lib.SYMBOLS
        assert hasattr(_lib.load(), name)
