"""CPU: which sampler takes which model wrapper, as one table.

Every sampler entry point is called with a bare MDM, a ClassifierFreeSampleModel and each feature wrapper
(HandshakeSampleModel, JointControlSampleModel, MultiPromptSampleModel), each of them once more behind
respace._WrappedModel, and a valid y.  A supported pair gets as far as the engine, which on the CPU is MDM.engine()'s
RuntimeError; an unsupported pair raises the sampler's refusal.  The type and the exact message of the first exception
are checked.  Then the wrapper constructors, _chain_plan and engine_for are given what they must refuse."""
import functools
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm.diffusion.respace import _WrappedModel
from b200mdm.model.mdm import engine_for
from b200mdm.utils.sampler_util import _chain_plan
from conftest import default_args

B, T, K = 2, 24, 2
ENGINE = "b200mdm runs on an H100 only (model is on cpu); move it with model.to('cuda'). There is no CPU / eager fallback."

# sampler family: the feature-wrapper kinds it refuses with NotImplementedError("<family> with <wrapper> is not implemented")
REFUSED = {"DDPM / DDIM": (), "PLMS": ("joint",), "DPM-Solver++": ("joint",), "DDIM inversion": ("handshake", "joint"),
           "p_mean_variance": ("joint",), "The variational bound": ("handshake", "joint", "multi")}
WRAPPER = {"handshake": "HandshakeSampleModel", "joint": "joint-position control (JointControlSampleModel)",
           "multi": "multi-prompt guidance (MultiPromptSampleModel)"}
KIND = {"mdm": None, "cfg": None, "handshake": "handshake", "joint": "joint", "multi": "multi"}


@functools.lru_cache(maxsize=None)
def _built(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def _dip():
    return _built(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)[0]


@functools.lru_cache(maxsize=None)
def _models():
    mdm, diffusion = _built()
    cfg = b200mdm.ClassifierFreeSampleModel(mdm)
    models = {"mdm": mdm, "cfg": cfg, "handshake": b200mdm.HandshakeSampleModel(cfg, 2),
              "joint": b200mdm.JointControlSampleModel(cfg, torch.zeros(263), torch.ones(263), 1e-3, 4),
              "multi": b200mdm.MultiPromptSampleModel(mdm)}
    for name in list(models):
        models["wrapped_" + name] = _WrappedModel(models[name], diffusion.timestep_map, False, diffusion.num_timesteps)
    return models, diffusion


def _y(**extra):
    return dict(text_embed=torch.zeros(1, B, 512), scale=torch.ones(B), lengths=torch.full((B,), T),
                mask=torch.ones(B, 1, 1, T, dtype=torch.bool), joint_target=torch.zeros(B, 22, 3, T),
                joint_weight=torch.ones(B, 22, T), prompt_embed=torch.zeros(K, B, 512),
                prompt_weight=torch.ones(B, K, 1, 1), **extra)


def _entry_points(d):
    """name: (sampler family, call(model))"""
    shape, x, t = (B, 263, 1, T), torch.zeros(B, 263, 1, T), torch.ones(B, dtype=torch.long)
    kw = lambda: {"y": _y()}                                                            # noqa: E731
    ar = b200mdm.AutoRegressiveSampler(SimpleNamespace(pred_len=12, context_len=12), d.p_sample_loop, required_frames=T)
    windows = dict(motion_start=torch.tensor([True, False]))
    return {
        "p_sample_loop": ("DDPM / DDIM", lambda m: d.p_sample_loop(m, shape, model_kwargs=kw())),
        "p_sample_loop_progressive": ("DDPM / DDIM", lambda m: next(d.p_sample_loop_progressive(m, shape, model_kwargs=kw()))),
        "p_sample": ("DDPM / DDIM", lambda m: d.p_sample(m, x, t, model_kwargs=kw())),
        "ddim_sample_loop": ("DDPM / DDIM", lambda m: d.ddim_sample_loop(m, shape, model_kwargs=kw())),
        "ddim_sample_loop_progressive": ("DDPM / DDIM",
                                         lambda m: next(d.ddim_sample_loop_progressive(m, shape, model_kwargs=kw()))),
        "ddim_sample": ("DDPM / DDIM", lambda m: d.ddim_sample(m, x, t, model_kwargs=kw())),
        "plms_sample_loop": ("PLMS", lambda m: d.plms_sample_loop(m, shape, model_kwargs=kw())),
        "plms_sample_loop_progressive": ("PLMS", lambda m: next(d.plms_sample_loop_progressive(m, shape, model_kwargs=kw()))),
        "plms_sample": ("PLMS", lambda m: d.plms_sample(m, x, t, model_kwargs=kw())),
        "dpm_solver_sample_loop": ("DPM-Solver++", lambda m: d.dpm_solver_sample_loop(m, shape, model_kwargs=kw())),
        "dpm_solver_sample_loop_progressive": ("DPM-Solver++",
                                               lambda m: next(d.dpm_solver_sample_loop_progressive(m, shape, model_kwargs=kw()))),
        "ddim_reverse_sample": ("DDIM inversion", lambda m: d.ddim_reverse_sample(m, x, t, model_kwargs=kw())),
        "ddim_reverse_sample_loop": ("DDIM inversion", lambda m: d.ddim_reverse_sample_loop(m, x, model_kwargs=kw())),
        "ddim_reverse_sample_loop_progressive": ("DDIM inversion",
                                                 lambda m: next(d.ddim_reverse_sample_loop_progressive(m, x, model_kwargs=kw()))),
        "p_mean_variance": ("p_mean_variance", lambda m: d.p_mean_variance(m, x, t, model_kwargs=kw())),
        "calc_bpd_loop": ("The variational bound", lambda m: d.calc_bpd_loop(m, x, model_kwargs=kw())),
        "AutoRegressiveSampler.sample": (
            "autoregressive", lambda m: ar.sample(m, shape, model_kwargs={"y": _y(prefix=torch.zeros(B, 263, 1, 12))})),
        "refine_transitions": (
            "transitions", lambda m: b200mdm.refine_transitions(d.ddim_sample_loop, m, x, {"y": _y(**windows)}, 2, 3, 2)),
    }


def _expected(family, kind):
    if kind is None:
        return RuntimeError, ENGINE
    if family == "autoregressive":
        if kind == "joint":
            return NotImplementedError, "the autoregressive chain is not implemented with joint-position control"
        return RuntimeError, ENGINE
    if family == "transitions":
        return TypeError, {
            "joint": "refine_transitions is not implemented with joint-position control (JointControlSampleModel)",
            "multi": "refine_transitions is not implemented with multi-prompt guidance (MultiPromptSampleModel)",
            "handshake": "refine_transitions runs the plain model: pass the model a HandshakeSampleModel wraps, not the "
                         "wrapper"}[kind]
    if kind in REFUSED[family]:
        return NotImplementedError, "%s with %s is not implemented" % (family, WRAPPER[kind])
    return RuntimeError, ENGINE


def _raised(call):
    with pytest.raises(Exception) as info:
        call()
    return type(info.value), str(info.value)


ENTRY_POINTS = list(_entry_points(_models()[1]))


@pytest.mark.parametrize("wrapped", [False, True])
@pytest.mark.parametrize("wrapper", list(KIND))
@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_support_matrix(entry, wrapper, wrapped):
    models, diffusion = _models()
    family, call = _entry_points(diffusion)[entry]
    model = models[("wrapped_" if wrapped else "") + wrapper]
    assert _raised(lambda: call(model)) == _expected(family, KIND[wrapper])


@pytest.mark.parametrize("wrapped", [False, True])
def test_autoregressive_chain_of_a_guided_dip_model(wrapped):
    dip = _dip()
    _, diffusion = _models()
    model = b200mdm.ClassifierFreeSampleModel(dip)
    if wrapped:
        model = _WrappedModel(model, diffusion.timestep_map, False, diffusion.num_timesteps)
    y = {"text_embed": (torch.zeros(5, B, 768), torch.zeros(B, 5, dtype=torch.bool)), "scale": torch.ones(B),
         "prefix": torch.zeros(B, 263, 1, 20)}
    ar = b200mdm.AutoRegressiveSampler(SimpleNamespace(pred_len=40, context_len=20), diffusion.p_sample_loop,
                                       required_frames=80)
    assert _raised(lambda: ar.sample(model, (B, 263, 1, 60), model_kwargs={"y": y})) == (RuntimeError, ENGINE)


def test_refine_transitions_refuses_dip_and_foreign_models():
    _, diffusion = _models()
    x = torch.zeros(B, 263, 1, T)
    kw = {"y": _y(motion_start=torch.tensor([True, False]))}
    for model in (_dip(), b200mdm.ClassifierFreeSampleModel(_dip())):
        assert _raised(lambda: b200mdm.refine_transitions(diffusion.ddim_sample_loop, model, x, kw, 2, 3, 2)) == (
            NotImplementedError, "transitions are not implemented for prefix-completion (DiP) models")
    foreign = SimpleNamespace(model=_models()[0]["mdm"])
    assert _raised(lambda: b200mdm.refine_transitions(diffusion.ddim_sample_loop, foreign, x, kw, 2, 3, 2)) == (
        TypeError, "HandshakeSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)" % type(foreign))


def _constructor_cases():
    models, diffusion = _models()
    mdm, cfg = models["mdm"], models["cfg"]
    stats = (torch.zeros(263), torch.ones(263), 1e-3, 4)
    dip = _dip()
    hs = lambda m: b200mdm.HandshakeSampleModel(m, 2)                                   # noqa: E731
    jc = lambda m: b200mdm.JointControlSampleModel(m, *stats)                           # noqa: E731
    mp = b200mdm.MultiPromptSampleModel
    hs_type = "HandshakeSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)"
    jc_type = "JointControlSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)"
    mp_type = "MultiPromptSampleModel wraps a b200mdm MDM (got %r)"
    cases = []
    for name, make, type_msg, dip_msg, inner in (
            ("HandshakeSampleModel", hs, hs_type, "handshakes are not implemented for prefix-completion (DiP) models", cfg),
            ("JointControlSampleModel", jc, jc_type,
             "joint-position control is not implemented for prefix-completion (DiP) models", cfg),
            ("MultiPromptSampleModel", mp, mp_type,
             "multi-prompt guidance is not implemented for prefix-completion (DiP) models", mdm)):
        for what, bad in (("wrapped", _WrappedModel(inner, diffusion.timestep_map, False, diffusion.num_timesteps)),
                          ("foreign", SimpleNamespace(model=mdm)), ("handshake", models["handshake"]),
                          ("joint", models["joint"]), ("multi", models["multi"])):
            cases.append(("%s-%s" % (name, what), make, bad, TypeError, type_msg % type(bad)))
        cases.append(("%s-dip" % name, make, dip, NotImplementedError, dip_msg))
    cases.append(("MultiPromptSampleModel-cfg", mp, cfg, TypeError, mp_type % type(cfg)))
    guided_dip = b200mdm.ClassifierFreeSampleModel(dip)
    cases.append(("HandshakeSampleModel-guided_dip", hs, guided_dip, NotImplementedError,
                  "handshakes are not implemented for prefix-completion (DiP) models"))
    cases.append(("JointControlSampleModel-guided_dip", jc, guided_dip, NotImplementedError,
                  "joint-position control is not implemented for prefix-completion (DiP) models"))
    return {case[0]: case[1:] for case in cases}


@pytest.mark.parametrize("case", list(_constructor_cases()))
def test_wrapper_constructors_refuse(case):
    make, model, exc, msg = _constructor_cases()[case]
    assert _raised(lambda: make(model)) == (exc, msg)


def test_chain_plan_takes_a_dip_model_and_its_guidance_only():
    models, diffusion = _models()
    dip = _dip()
    kargs = {"model_kwargs": {"y": {"prefix": torch.zeros(B, 263, 1, 20)}}}
    shape = (B, 263, 1, 40)
    for model in (dip, b200mdm.ClassifierFreeSampleModel(dip)):
        assert _chain_plan(diffusion.p_sample_loop, model, shape, 2, kargs) is not None
    for model in (_WrappedModel(b200mdm.ClassifierFreeSampleModel(dip), diffusion.timestep_map, False, diffusion.num_timesteps),
                  _WrappedModel(dip, diffusion.timestep_map, False, diffusion.num_timesteps),
                  models["cfg"], models["mdm"], SimpleNamespace(model=dip)):
        assert _chain_plan(diffusion.p_sample_loop, model, shape, 2, kargs) is None


def test_engine_for_refuses_what_it_cannot_unwrap():
    models, _ = _models()
    cfg_of_cfg = b200mdm.ClassifierFreeSampleModel(models["cfg"])
    assert _raised(lambda: engine_for(cfg_of_cfg)) == (
        TypeError, "ClassifierFreeSampleModel must wrap a b200mdm MDM (got %r)" % type(models["cfg"]))
    foreign = SimpleNamespace(model=models["mdm"])
    assert _raised(lambda: engine_for(foreign)) == (
        TypeError, "b200mdm diffusion objects drive b200mdm.MDM or b200mdm.ClassifierFreeSampleModel only (got %r); "
                   "wrap the model with the classes of this package" % type(foreign))
    for name, model in models.items():
        assert _raised(lambda: engine_for(model)) == (RuntimeError, ENGINE), name
