"""CPU: the sampling extensions on the BERT decoder with context_len 0 (humanml_trans_dec_512_bert).

  * all four wrappers accept it, and a context_len = 20 DiP still raises NotImplementedError;
  * the token-pair y['prompt_embed'] and y['prompt_text'] are checked before any engine work, y untouched;
  * parallel.shard_model_kwargs slices the pairs, and the (tokens, mask) text_embed of chained windows;
  * the transitions' conditioning gathers token columns and mask rows as a hand-built gather does;
  * the decoder multi-prompt oracle at K = 1 is cfg_denoise_dec;
  * b200mdm_set_cond_multi_tokens: its argument checks before any CUDA call, and its place in the header."""
import ctypes
import os
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from b200mdm.utils import sampler_util as su
from conftest import ROOT, default_args, rel_err
import bert_dec_oracle as bdo
from oracle import double_take_oracle as dt
from oracle import mdm_oracle as mo

syn = b200mdm.synthetic


def _bert(ctx=0):
    return b200mdm.create_model_and_diffusion(
        default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert", context_len=ctx,
                     pred_len=40 if ctx else 0), SimpleNamespace(dataset=SimpleNamespace()))


def test_wrappers_accept_the_bert_decoder_and_refuse_dip():
    mean, std = torch.zeros(263), torch.ones(263)
    model, diffusion = _bert()
    assert model.is_dip and not model.is_prefix_comp
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    assert b200mdm.HandshakeSampleModel(cfg, 4).handshake_size == 4
    assert b200mdm.JointControlSampleModel(cfg, mean, std, 1e-3, 2).n_joints == 22
    assert b200mdm.MultiPromptSampleModel(model).kind == "multi"
    # refine_transitions: single-window motions need no engine call, so acceptance shows on the CPU
    windows = torch.randn(2, 263, 1, 24)
    y = {"lengths": torch.tensor([24, 20]), "motion_start": torch.tensor([True, True])}
    motions = b200mdm.refine_transitions(diffusion.p_sample_loop, cfg, windows, {"y": y}, 2, 2, 1)
    assert [m.shape[-1] for m in motions] == [24, 20]
    dip, ddiff = _bert(ctx=20)
    assert dip.is_dip and dip.is_prefix_comp
    dcfg = b200mdm.ClassifierFreeSampleModel(dip)
    for make in (lambda: b200mdm.HandshakeSampleModel(dcfg, 4),
                 lambda: b200mdm.JointControlSampleModel(dcfg, mean, std, 1e-3, 2),
                 lambda: b200mdm.MultiPromptSampleModel(dip),
                 lambda: b200mdm.refine_transitions(ddiff.p_sample_loop, dcfg, windows, {"y": y}, 2, 2, 1)):
        with pytest.raises(NotImplementedError):
            make()


def test_token_prompt_validation():
    model, diffusion = _bert()
    mp = b200mdm.MultiPromptSampleModel(model)
    B, K, T = 2, 2, 24
    x = torch.zeros(B, 263, 1, T)
    t = torch.zeros(B, dtype=torch.long)
    pairs = [(torch.zeros(5, B, 768), torch.zeros(B, 5, dtype=torch.bool)),
             (torch.zeros(70, B, 768), torch.zeros(B, 70, dtype=torch.bool))]
    y = {"prompt_embed": pairs, "prompt_weight": torch.ones(B, K, 1, 1), "lengths": torch.tensor([24, 7])}
    e, a, w = mp.prompts(y, x.shape)
    assert a is None and len(e) == K and all(p is q for p, q in zip(e, pairs))
    tok, msk = pairs[0]
    snapshot = dict(y)
    for bad in (torch.zeros(K, B, 768), pairs[:1], pairs + pairs[:1], [tok, pairs[1]], [(tok,), pairs[1]],
                [(tok.double()[..., :767], msk), pairs[1]], [(tok[:, :1], msk), pairs[1]],
                [(tok.long(), msk), pairs[1]], [(tok[:, 0], msk), pairs[1]], [(tok[:0], msk[:, :0]), pairs[1]],
                [(torch.zeros(513, B, 768), torch.zeros(B, 513, dtype=torch.bool)), pairs[1]],
                [(tok, msk[:, :4]), pairs[1]], [(tok, msk.float()), pairs[1]], [(tok, None), pairs[1]]):
        yy = dict(y, prompt_embed=bad)
        for call in (lambda: mp.prompts(yy, x.shape),
                     lambda: diffusion.p_sample_loop(mp, x.shape, model_kwargs={"y": yy}),
                     lambda: mp(x, t, y=yy)):
            with pytest.raises(ValueError):
                call()
        assert yy["prompt_embed"] is bad
    for bad in ([["a", "b"], ["c"]], ["ab", "cd"], [["a", "b"]]):
        yy = {"prompt_text": bad, "prompt_weight": torch.ones(B, K, 1, 1)}
        with pytest.raises(ValueError):
            diffusion.p_sample_loop(mp, x.shape, model_kwargs={"y": yy})
        assert "prompt_embed" not in yy
    assert y.keys() == snapshot.keys() and all(y[k] is snapshot[k] for k in y)
    # y['prompt_text'] is encoded one prompt column at a time into K pairs
    seen = []

    def encode(texts):
        seen.append(list(texts))
        n = len(seen) + 3
        return torch.zeros(n, len(texts), 768), torch.zeros(len(texts), n, dtype=torch.bool)
    mp.model.encode_text = encode
    enc = mp.encode_prompts([["a0", "b0"], ["a1", "b1"]])
    assert seen == [["a0", "a1"], ["b0", "b1"]] and [p[0].shape[0] for p in enc] == [4, 5]


def test_shard_model_kwargs_slices_token_pairs():
    B = 6
    pairs = [(torch.randn(9, B, 768), torch.rand(B, 9) < 0.3), (torch.randn(70, B, 768), torch.rand(B, 70) < 0.3)]
    te = (torch.randn(12, B, 768), torch.rand(B, 12) < 0.3)
    ms = torch.tensor([True, False, True, False, False, True])
    y = {"prompt_embed": pairs, "text_embed": te, "motion_start": ms, "lengths": torch.arange(B)}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    for (t, m), (pt, pm) in zip(pairs, part["prompt_embed"]):
        assert torch.equal(pt, t[:, 2:5]) and torch.equal(pm, m[2:5])
    assert torch.equal(part["text_embed"][0], te[0][:, 2:5]) and torch.equal(part["text_embed"][1], te[1][2:5])
    assert torch.equal(part["motion_start"], ms[2:5]) and torch.equal(part["lengths"], y["lengths"][2:5])
    with pytest.raises(ValueError):
        parallel.shard_model_kwargs({"y": y}, 0, 4)                  # window 4 continues window 3


def test_transition_y_gathers_tokens_and_masks():
    B, Mt, T, h, m = 5, 11, 30, 3, 2
    ln = torch.tensor([30, 28, 30, 30, 25])
    ms = torch.tensor([True, False, False, True, False])
    tok, msk = torch.randn(Mt, B, 768), torch.rand(B, Mt) < 0.4
    scale = torch.rand(B)
    y = {"text_embed": (tok, msk), "scale": scale, "lengths": ln, "motion_start": ms}
    later = [1, 2, 4]                                                # the later window of every transition
    want_tok = torch.stack([tok[:, b] for b in later], 1)
    want_msk = torch.stack([msk[b] for b in later], 0)
    lay = b200mdm.transition_layout(B, T, h, m, ln, ms)
    assert lay["pairs"][:, 1].tolist() == later
    got = su._transition_y(y, lay["pairs"][:, 1], 2 * m + h, "cpu")
    assert torch.equal(got["text_embed"][0], want_tok) and torch.equal(got["text_embed"][1], want_msk)
    assert torch.equal(got["scale"], scale[later])
    x_init = dt.gather(torch.randn(B, 263, 1, T), ln, ms, h, m)
    ref = bdo.transition_y(y, ln, ms, h, m, x_init)
    assert torch.equal(ref["text_embed"][0], want_tok) and torch.equal(ref["text_embed"][1], want_msk)
    # a single prompt for the whole batch stays shared
    one = (tok[:, :1], msk[:1])
    got = su._transition_y(dict(y, text_embed=one), lay["pairs"][:, 1], 2 * m + h, "cpu")
    assert got["text_embed"][0] is one[0] and got["text_embed"][1] is one[1]


def test_dec_oracle_k1_is_cfg():
    L, B, T, Mt = 2, 3, 16, 9
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=768, seed=3)
    inp = syn.synthetic_inputs(B, nframes=T, steps=0, seed=4, lengths=[16, 9, 2], scale=torch.tensor([2.5, 1.0, 7.5]))
    enc, tmask, _ = syn.synthetic_dip_inputs(B, Mt, 0, seed=5)
    tmask[:] = False
    tmask[1, 4:] = True
    W = mo.OracleWeights(sd, L)
    x, sc, ln = inp["tape"][0], inp["scale"], inp["lengths"]
    cfg = mo.cfg_denoise_dec(W, x, 7, enc, tmask, torch.zeros(B, 263, 1, 0), sc, ln)
    got = bdo.dec_denoiser(W, list(range(10)), [(enc, tmask)], sc.view(B, 1, 1, 1), ln)(x, 7)
    assert rel_err(got, cfg) < 1e-6


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    mask = (ctypes.c_uint8 * 16)()
    assert lib.b200mdm_set_cond_multi_tokens(None, 2, 24, 2, buf, mask, 4, None, None) == _lib.EINVAL
    assert b"null" in lib.b200mdm_last_error()
    header = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    assert "int b200mdm_set_cond_multi_tokens(" in header
    assert "b200mdm_set_cond_multi_tokens" in _lib.SYMBOLS
