"""CPU: host-side boundary -- the C-ABI library loads and exports every symbol include/b200mdm.h declares, the
Python mirror keeps the reference's API surface, and the product refuses to run without a GPU (no fallback)."""
import ctypes
import os
import re
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from conftest import ROOT, default_args


def test_header_symbols_exported():
    from b200mdm import _lib
    hdr = open(os.path.join(ROOT, "include", "b200mdm.h")).read()
    declared = sorted(set(re.findall(r"\b(b200mdm_[a-z0-9_]+)\s*\(", hdr)))
    assert declared, "no declarations parsed"
    assert sorted(_lib.SYMBOLS) == declared
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.b200mdm_version() >= 1
    assert ctypes.sizeof(_lib.Config) == 20 * 4


def test_api_surface_matches_reference():
    args = default_args(layers=2)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    # attributes the reference's callers read (sample/generate.py:95-98,161-171; sampler_util.py:16-25)
    for a in ["njoints", "nfeats", "data_rep", "cond_mode", "cond_mask_prob", "translation", "rot2xyz", "encode_text",
              "text_encoder_type", "all_goal_joint_names", "parameters", "to", "eval", "train"]:
        assert hasattr(model, a), a
    assert (model.njoints, model.nfeats, model.data_rep, model.cond_mode) == (263, 1, "hml_vec", "text")
    for a in ["num_timesteps", "timestep_map", "original_num_steps", "betas", "alphas_cumprod", "posterior_variance",
              "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2", "model_mean_type",
              "model_var_type", "p_sample_loop", "p_sample_loop_progressive", "ddim_sample_loop",
              "ddim_sample_loop_progressive", "p_sample", "ddim_sample", "q_sample"]:
        assert hasattr(diffusion, a), a
    assert diffusion.num_timesteps == 50 and diffusion.timestep_map == list(range(50))
    # reference state_dict keys / shapes (SURVEY.md A.4) load through the reference-style loader
    sd = b200mdm.synthetic_state_dict(num_layers=2)
    assert set(sd) == set(model.state_dict())
    for k, v in model.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    sd["sequence_pos_encoder.pe"] = torch.zeros(5000, 1, 512)
    sd["embed_timestep.sequence_pos_encoder.pe"] = torch.zeros(5000, 1, 512)
    b200mdm.load_model_wo_clip(model, sd)
    assert torch.equal(model.state_dict()["output_process.poseFinal.bias"], sd["output_process.poseFinal.bias"])
    with pytest.raises(AssertionError):
        b200mdm.load_model_wo_clip(model, dict(sd, bogus=torch.zeros(1)))
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    assert cfg.njoints == 263 and cfg.cond_mask_prob == 0.1 and cfg.all_goal_joint_names[0] == "pelvis"
    m0, _ = b200mdm.create_model_and_diffusion(default_args(layers=1, cond_mask_prob=0.0), SimpleNamespace(dataset=SimpleNamespace()))
    with pytest.raises(AssertionError):
        b200mdm.ClassifierFreeSampleModel(m0)


def test_unsupported_configs_raise():
    for over in (dict(arch="gru"), dict(arch="trans_dec", text_encoder_type="clip"),
                 dict(arch="trans_dec", text_encoder_type="bert", emb_trans_dec=True),
                 dict(arch="trans_enc", context_len=20, pred_len=40)):
        with pytest.raises(NotImplementedError):
            b200mdm.create_model_and_diffusion(default_args(layers=1, **over), SimpleNamespace(dataset=SimpleNamespace()))


def test_dip_model_keys_match_reference_layout():
    """trans_dec / BERT (DiP): parameter names and shapes of nn.TransformerDecoderLayer (model/mdm.py:87-96,110-119)."""
    args = default_args(layers=2, arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    model, _ = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    assert model.clip_dim == 768 and model.is_prefix_comp and model.total_len == 60
    sd = model.state_dict()
    want = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=4)
    assert set(sd.keys()) == set(want.keys())
    for k, v in want.items():
        assert tuple(sd[k].shape) == tuple(v.shape), k
    assert "seqTransDecoder.layers.1.multihead_attn.in_proj_weight" in sd and "seqTransDecoder.layers.0.norm3.bias" in sd
    b200mdm.load_model_wo_clip(model, want)


def test_autoregressive_sampler_chunks():
    """AutoRegressiveSampler (utils/sampler_util.py:41-81): chunk count, prefix hand-over, cropping -- with a stub
    sample_fn, no GPU."""
    args = SimpleNamespace(pred_len=40, context_len=20, autoregressive_include_prefix=False)
    seen = []

    def sample_fn(model, shape, **kw):
        y = kw["model_kwargs"]["y"]
        seen.append((tuple(shape), y["prefix"].clone()))
        return torch.full(shape, float(len(seen))) + torch.arange(shape[-1]).float() / 100

    prefix = torch.zeros(2, 263, 1, 20)
    y = {"prefix": prefix, "text": ["a", "b"]}
    out = b200mdm.AutoRegressiveSampler(args, sample_fn, required_frames=196).sample(None, (2, 263, 1, 196), model_kwargs={"y": y})
    assert out.shape == (2, 263, 1, 196) and len(seen) == 5
    assert all(s[0] == (2, 263, 1, 40) for s in seen)
    assert torch.equal(seen[0][1], prefix) and y["prefix"] is prefix
    assert torch.equal(seen[2][1], torch.full((2, 263, 1, 20), 2.0) + torch.arange(20, 40).float() / 100)
    assert float(out[0, 0, 0, 0]) == 1.0 and abs(float(out[0, 0, 0, 195]) - 5.35) < 1e-6
    args.autoregressive_include_prefix = True
    out = b200mdm.AutoRegressiveSampler(args, sample_fn, required_frames=100).sample(None, (2, 263, 1, 100), model_kwargs={"y": y})
    assert out.shape == (2, 263, 1, 100) and torch.equal(out[..., :20], prefix)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=1), SimpleNamespace(dataset=SimpleNamespace()))
    x = torch.zeros(1, 263, 1, 8)
    y = {"text_embed": torch.zeros(1, 1, 512), "mask": torch.ones(1, 1, 1, 8, dtype=torch.bool), "lengths": torch.tensor([8])}
    with pytest.raises(RuntimeError):
        model(x, torch.zeros(1, dtype=torch.long), y=y)
    with pytest.raises(RuntimeError):
        diffusion.p_sample_loop(model, (1, 263, 1, 8), clip_denoised=False, model_kwargs={"y": y})


def test_c_abi_error_contract_without_gpu():
    """include/b200mdm.h: every entry point returns 0 or a negative B200MDM_E* code and leaves a message in
    b200mdm_last_error(); argument validation happens before any CUDA call, so this runs without a GPU."""
    import ctypes
    from b200mdm import _lib
    lib = _lib.load()
    lib.b200mdm_last_error.restype = ctypes.c_char_p
    h = ctypes.c_void_p()
    assert lib.b200mdm_create(None, ctypes.byref(h)) < 0 and b"null" in lib.b200mdm_last_error()
    cfg = _lib.Config(arch=7, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, njoints=263, nfeats=1, cond_mode=_lib.COND_TEXT,
                      cond_dim=512, num_actions=1, mask_frames=1, pos_embed_max_len=5000, temb_rows=1000)
    assert lib.b200mdm_create(ctypes.byref(cfg), ctypes.byref(h)) < 0 and b"arch 7" in lib.b200mdm_last_error()
    cfg.arch, cfg.latent_dim = _lib.ARCH["trans_enc"], 256
    assert lib.b200mdm_create(ctypes.byref(cfg), ctypes.byref(h)) < 0 and b"latent_dim 512" in lib.b200mdm_last_error()
    cfg.latent_dim, cfg.arch, cfg.cond_mode = 512, _lib.ARCH["trans_dec"], _lib.COND_ACTION
    assert lib.b200mdm_create(ctypes.byref(cfg), ctypes.byref(h)) < 0 and b"trans_dec" in lib.b200mdm_last_error()
    assert not h.value
    # post-processing entry point: pointer / shape checks
    buf = (ctypes.c_float * 4)()
    assert lib.b200mdm_recover_from_ric(None, 0, 0, 0, None, None, buf, 0, 0, 0, 1, 1, 22, None) < 0
    assert lib.b200mdm_recover_from_ric(buf, 1, 1, 1, buf, None, buf, 1, 1, 1, 1, 1, 22, None) < 0 and b"mean and std" in lib.b200mdm_last_error()
    assert lib.b200mdm_recover_from_ric(buf, 1, 1, 1, None, None, buf, 1, 1, 1, 1, 100000, 22, None) < 0 and b"frames" in lib.b200mdm_last_error()
    # kernel-test hook of the projection GEMM: block_n is 128 (128 x 128 tiles) or the call is refused
    for bn in (512, 513, 64, 0):
        assert lib.b200mdm_test_gemm_f16(buf, buf, buf, buf, 128, 128, 64, 0, bn, None) == _lib.EINVAL
        assert b"block_n must be 128" in lib.b200mdm_last_error()
    for fn in (lib.b200mdm_set_cond_dec, lib.b200mdm_set_prefix):
        assert fn.argtypes is not None
    assert lib.b200mdm_set_prefix(None, None, None) < 0
    assert lib.b200mdm_version() >= 1


def test_alias_submodules_are_the_same_objects():
    """ADVICE r1: `from b200mdm.utils.sampler_util import X` must hand out the package's own class object (a second copy of
    the module tree made engine_for() unwrap a guidance wrapper down to the bare denoiser, silently dropping CFG)."""
    import importlib
    import b200mdm
    from b200mdm.utils.sampler_util import ClassifierFreeSampleModel as A
    from b200mdm.diffusion.respace import SpacedDiffusion as S_
    import b200mdm.model.mdm as m1
    assert A is b200mdm.ClassifierFreeSampleModel and S_ is b200mdm.SpacedDiffusion
    assert m1 is importlib.import_module("motion-diffusion-model_b200.model.mdm")


def test_engine_for_rejects_foreign_wrappers():
    """A wrapper class this package does not know (here: something with a `.model` attribute) is not looked through."""
    from types import SimpleNamespace
    import pytest
    import b200mdm
    from b200mdm.model.mdm import engine_for
    model, _ = b200mdm.create_model_and_diffusion(default_args(layers=1), SimpleNamespace(dataset=SimpleNamespace()))
    with pytest.raises(TypeError):
        engine_for(SimpleNamespace(model=model))
