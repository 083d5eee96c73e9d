"""CPU: the CLIP-conditioned decoder with a timestep token (arch='trans_dec', text_encoder_type='clip',
emb_trans_dec=True) -- the fp32 oracle against the reference's fixtures, the host model's parameter layout, the C
config layout, the configurations that still raise and the C-ABI rejections that happen before any CUDA call."""
import ctypes
import importlib
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from conftest import ROOT, default_args, rel_err
from oracle import dec_emb_oracle as deo, mdm_oracle as mo, schedule_oracle as so, target_oracle as to

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")
L, STEPS, B, T = 2, 4, 3, 24


def _small():
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=9)
    inp = syn.synthetic_inputs(B, nframes=T, steps=STEPS, seed=15, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 7.5]))
    return sd, inp


def _inpaint(g):
    motion = torch.from_numpy(g["inpaint_motion"])
    m = torch.zeros(motion.shape, dtype=torch.bool)
    m[..., :8] = True
    return m, motion


def test_oracle_matches_dec_emb_small(golden):
    g = golden("dec_emb_small.npz")
    sd, inp = _small()
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", STEPS))
    x, te, ln, sc = inp["tape"][0], inp["text_embed"], inp["lengths"], inp["scale"]
    with torch.no_grad():
        got = {"fwd_cond": deo.denoise_dec_emb(W, x, 2, te, ln),
               "fwd_uncond": deo.denoise_dec_emb(W, x, 2, te, ln, uncond=True),
               "fwd_cfg": deo.cfg_denoise_dec_emb(W, x, 2, te, sc, ln),
               "nomask_fwd_cfg": deo.cfg_denoise_dec_emb(W, x, 2, te, sc, ln, mask_frames=False)}
        f = deo.denoiser(W, list(range(STEPS)), te, sc, ln)
        got["ddpm"] = deo.sample_loop(f, tabs, inp["tape"])
        got["ddim_eta0"] = deo.sample_loop(f, tabs, inp["tape"], sampler="ddim")
        got["ddpm_inpaint"] = deo.sample_loop(f, tabs, inp["tape"], inpaint=_inpaint(g))
        got["nomask_ddpm"] = deo.sample_loop(deo.denoiser(W, list(range(STEPS)), te, sc, ln, mask_frames=False), tabs, inp["tape"])
        sdt = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=9, target_encoder="single")
        Wt = mo.OracleWeights(sdt, L)
        tg = syn.synthetic_target_inputs(B, seed=5)
        valid = to.validity(syn.HML_TARGET_JOINTS, tg["target_joint_names"], tg["is_heading"])
        gt = to.target_embedding(Wt, "single", tg["target_cond"], valid)
        got["target_g"] = gt
        got["target_fwd_cfg"] = deo.cfg_denoise_dec_emb(Wt, x, 2, te, sc, ln, g=gt)
        got["target_ddpm"] = deo.sample_loop(deo.denoiser(Wt, list(range(STEPS)), te, sc, ln, g=gt), tabs, inp["tape"])
    for k, v in got.items():
        e = rel_err(v, g[k])
        print("%-16s %.2e" % (k, e))
        assert e < 2e-5, k
    # the target term and the key mask each change the result (the fixture would not catch their loss otherwise)
    assert rel_err(g["nomask_fwd_cfg"], g["fwd_cfg"]) > 1e-2 and rel_err(g["target_fwd_cfg"], g["fwd_cfg"]) > 1e-2


def test_oracle_matches_dec_emb_c1(golden):
    g = golden("dec_emb_c1.npz")
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=8, cond_dim=512, seed=0)
    inp = syn.synthetic_inputs(1, nframes=196, steps=50, seed=10)
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", 50))
    with torch.no_grad():
        out = deo.sample_loop(deo.denoiser(W, list(range(50)), inp["text_embed"], inp["scale"], inp["lengths"]), tabs, inp["tape"])
    e = rel_err(out, g["sample"])
    print("c1 decoder, 50 steps: %.2e" % e)
    assert e < 1e-4


def _dec_emb_args(**over):
    return default_args(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True, **over)


def test_model_keys_match_synthetic_and_reference():
    model, diffusion = b200mdm.create_model_and_diffusion(_dec_emb_args(layers=2), SimpleNamespace(dataset=SimpleNamespace()))
    assert model.clip_dim == 512 and model.emb_trans_dec and model.text_encoder_type == "clip"
    sd = model.state_dict()
    want = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=512, seed=3)
    assert set(sd) == set(want)
    for k, v in want.items():
        assert tuple(sd[k].shape) == tuple(v.shape), k
    assert tuple(sd["embed_text.weight"].shape) == (512, 512)
    b200mdm.load_model_wo_clip(model, want)
    from oracle import ref_harness as rh
    if not rh.available():
        return
    ref, _ = rh.build(rh.default_args(layers=2, arch="trans_dec", emb_trans_dec=True, text_encoder_type="clip"))
    rsd = {k: v for k, v in ref.state_dict().items() if not k.startswith("clip_model.") and "sequence_pos_encoder" not in k}
    assert set(rsd) == set(want)
    for k, v in rsd.items():
        assert tuple(v.shape) == tuple(want[k].shape), k


def test_old_args_without_text_encoder_type_load_clip():
    """An args.json written before the BERT option has no text_encoder_type; the reference then loads CLIP."""
    args = _dec_emb_args(layers=1)
    del args.text_encoder_type
    model, _ = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    assert model.text_encoder_type == "clip" and model.clip_dim == 512


def test_config_field_offsets():
    assert ctypes.sizeof(_lib.Config) == 20 * 4
    assert _lib.Config.emb_trans_dec.offset == 17 * 4 and _lib.Config.dec_memory.offset == 18 * 4
    assert _lib.Config.reserved.offset == 19 * 4
    assert _lib.Config.target_joints.offset == 16 * 4


@pytest.mark.parametrize("over", [
    dict(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=False),
    dict(arch="trans_dec", text_encoder_type="bert", emb_trans_dec=True),
    dict(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True, unconstrained=True),
    dict(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True, context_len=20, pred_len=40),
])
def test_other_decoder_configs_still_raise(over):
    with pytest.raises(NotImplementedError):
        b200mdm.create_model_and_diffusion(default_args(layers=1, **over), SimpleNamespace(dataset=SimpleNamespace()))


def test_trans_dec_with_action_raises():
    args = default_args(layers=1, arch="trans_dec", emb_trans_dec=True, dataset="humanact12", unconstrained=False)
    with pytest.raises(NotImplementedError):
        b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace(num_actions=12)))


def _cfg(**over):
    c = dict(arch=_lib.ARCH["trans_dec"], latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, njoints=263, nfeats=1,
             cond_mode=_lib.COND_TEXT, cond_dim=512, num_actions=1, mask_frames=1, pos_embed_max_len=5000, temb_rows=1000,
             emb_trans_dec=1, dec_memory=_lib.DEC_MEMORY_CLIP)
    c.update(over)
    return _lib.Config(**c)


@pytest.mark.parametrize("over, code, text", [
    (dict(emb_trans_dec=0), _lib.ENOTIMPL, b"emb_trans_dec"),                      # the plain CLIP decoder
    (dict(dec_memory=_lib.DEC_MEMORY_TOKENS, cond_dim=768), _lib.ENOTIMPL, b"emb_trans_dec"),   # BERT + timestep token
    (dict(context_len=20), _lib.ENOTIMPL, b"context_len"),
    (dict(cond_mode=_lib.COND_ACTION), _lib.ENOTIMPL, b"trans_dec"),
    (dict(dec_memory=2), _lib.EINVAL, b"dec_memory"),
    (dict(emb_trans_dec=3), _lib.EINVAL, b"emb_trans_dec"),
    (dict(arch=_lib.ARCH["trans_enc"]), _lib.EINVAL, b"trans_dec fields"),
])
def test_c_abi_rejections_before_any_cuda_call(over, code, text):
    lib = _lib.load()
    h = ctypes.c_void_p()
    cfg = _cfg(**over)
    assert lib.b200mdm_create(ctypes.byref(cfg), ctypes.byref(h)) == code
    assert text in lib.b200mdm_last_error() and not h.value


def test_test_hooks_reject_bad_arguments_without_gpu():
    lib = _lib.load()
    assert lib.b200mdm_test_cross_rows(None, 0, None, None) == _lib.EINVAL
    assert lib.b200mdm_test_row_bias_ln(None, None, None, None, 8, 4, None) == _lib.EINVAL
    assert lib.b200mdm_test_tap_bytes(None, 0) == _lib.EINVAL


def test_forward_taps_rejects_bad_arguments_without_gpu():
    """b200mdm_test_forward_taps validates its arguments before any CUDA call; the tap ids are the header's."""
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    ids = {m[0]: int(m[1]) for m in re.findall(r"#define B200MDM_TAP_([A-Z0-9_]+) (\d+)", hdr)}
    assert ids.pop("COUNT") == len(_lib.TAPS) and ids == {n: i for i, n in enumerate(_lib.TAPS)}
    buf = (ctypes.c_float * 4)()
    ts = (ctypes.c_int32 * 1)()
    taps = (ctypes.c_void_p * len(_lib.TAPS))()
    fn = lib.b200mdm_test_forward_taps
    assert fn(None, buf, ts, buf, 0, taps, len(_lib.TAPS), None) == _lib.EINVAL
    assert b"null" in lib.b200mdm_last_error()
    for x, t, out in ((None, ts, buf), (buf, None, buf), (buf, ts, None)):
        assert fn(None, x, t, out, 0, taps, 1, None) == _lib.EINVAL
