"""GPU: DiP's autoregressive chain as engine loops (AutoRegressiveSampler with p_sample_loop, ddim_sample_loop or
dpm_solver_sample_loop; DESIGN.md, "Autoregressive chain").

  * bit-identity (torch.equal) with the host chain -- reached through a non-eligible callable -- across samplers,
    guidance, static and per-chunk text, include_prefix, cropping, every noise source, target conditioning, inpainting,
    a respaced schedule, graph and eager launches, and a 200-token memory;
  * one engine across chains and plain loops against fresh engines; a Philox batch split against the whole batch;
  * one conditioning upload per chain, and a warmed-up chain that enqueues without a host synchronisation;
  * a small chain against the fp32 oracle chain, and the device chain against the unmodified reference's chain
    (tests/golden/dip_ar_small.npz);
  * the C ABI's rejections that need an engine."""
import ctypes
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import mdm_oracle as mo
from oracle import schedule_oracle as so

ga = importlib.import_module("oracle.gen_golden_ar_chain")

pytestmark = pytest.mark.gpu
L, CTX, PRED, STEPS, C = 2, 4, 8, 4, 768


class FakeBert:
    """A deterministic stand-in for the DistilBERT wrapper (model/mdm.py bert_encode_text): features seeded by the text,
    `mt` tokens, the first 1 + len(text) % mt present."""

    def __init__(self, mt):
        self.mt = mt

    def __call__(self, texts):
        enc = torch.stack([torch.randn(self.mt, C, generator=torch.Generator().manual_seed(sum(map(ord, t)) + 7))
                           for t in texts]).cuda()
        present = torch.zeros(len(texts), self.mt, dtype=torch.bool)
        for b, t in enumerate(texts):
            present[b, :1 + len(t) % self.mt] = True
        return enc, present.cuda()


def build(steps=STEPS, respacing=None, target=False, mt=6, ctx=CTX, pred=PRED, seed=21, dataset="humanml"):
    over = dict(layers=L, diffusion_steps=steps, arch="trans_dec", text_encoder_type="bert", context_len=ctx, pred_len=pred,
                dataset=dataset)
    if target:
        over.update(multi_target_cond=True, multi_encoder_type="multi", target_enc_layers=1)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=C, seed=seed,
                                      target_encoder="multi" if target else None, input_feats=251 if dataset == "kit" else 263)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    model.clip_model = FakeBert(mt)
    if respacing is not None:
        diffusion = rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(steps, respacing),
                                       betas=gd.get_named_beta_schedule("cosine", steps),
                                       model_mean_type=gd.ModelMeanType.START_X,
                                       model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    return model, diffusion, sd


def make_y(B, n_chunks, mt=6, ctx=CTX, pred=PRED, guided=True, text="static", seed=3, host_mask=False, njoints=263):
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, mt, ctx, njoints=njoints, seed=seed)
    y = dict(prefix=prefix.cuda(), mask=torch.ones(B, 1, 1, pred, dtype=torch.bool).cuda(),
             lengths=torch.tensor([pred] + [pred - 1 - b % 3 for b in range(1, B)]).cuda())
    if host_mask:
        y["lengths"] = y["lengths"].cpu()
    if guided:
        y["scale"] = torch.tensor([7.5, 2.0, 1.0, 3.0, 0.5, 4.0][:B]).cuda()
    if text == "static":
        y["text_embed"] = (enc.cuda(), tmask if host_mask else tmask.cuda())
    elif text == "encoded":
        y["text"] = ["a person walks %d" % b for b in range(B)]
    else:                                            # a prompt per chunk; the slices are replaced by encode_text
        y["text"] = [["prompt %d of sample %d" % (c, b) + "!" * (b + c) for c in range(n_chunks)] for b in range(B)]
        y["text_embed"] = (torch.zeros(mt, B, n_chunks, C).cuda(), torch.zeros(B, n_chunks, mt, dtype=torch.bool).cuda())
    return y


def host(fn):
    return lambda *a, **k: fn(*a, **k)


def run_both(model, diffusion, sampler, shape, required, include_prefix, seed=5, ctx=CTX, **kw):
    args = SimpleNamespace(pred_len=shape[-1], context_len=ctx, autoregressive_include_prefix=include_prefix)
    fn = getattr(diffusion, sampler)
    outs = []
    for f in (fn, host(fn)):
        torch.manual_seed(seed)
        torch.cuda.manual_seed(seed)
        outs.append(b200mdm.AutoRegressiveSampler(args, f, required_frames=required).sample(model, shape, **kw))
    torch.cuda.synchronize()
    return outs


CASES = {
    # name: (sampler, sampler kwargs, guided, text, include_prefix, required, noise form, use_graph)
    "ddpm_cfg_static": ("p_sample_loop", {}, True, "static", False, 30, "generator", True),
    "ddpm_cfg_dynamic_prefix": ("p_sample_loop", {}, True, "dynamic", True, 30, "generator", True),
    "ddpm_plain_encoded_tape_eager": ("p_sample_loop", {"clip_denoised": True}, False, "encoded", True, 27, "tape", False),
    "ddpm_cfg_philox": ("p_sample_loop", {}, True, "static", False, 32, "philox", True),
    "ddpm_cfg_xT_per_chunk": ("p_sample_loop", {}, True, "dynamic", False, 30, "x_T", True),
    "ddim0_cfg_dynamic": ("ddim_sample_loop", {"eta": 0.0}, True, "dynamic", True, 30, "generator", True),
    "ddim05_cfg_static_tape": ("ddim_sample_loop", {"eta": 0.5}, True, "static", False, 30, "tape", True),
    "ddim05_plain_philox_eager": ("ddim_sample_loop", {"eta": 0.5}, False, "static", True, 30, "philox", False),
    "dpm2_cfg_dynamic": ("dpm_solver_sample_loop", {"order": 2}, True, "dynamic", True, 30, "generator", True),
    "dpm2_cfg_philox": ("dpm_solver_sample_loop", {"order": 2}, True, "static", False, 30, "philox", True),
    "dpm1_plain_xT_eager": ("dpm_solver_sample_loop", {"order": 1}, False, "encoded", False, 25, "x_T", False),
}


def noise_kw(form, n_chunks, n_steps, shape):
    g = torch.Generator().manual_seed(99)
    if form == "tape":
        return dict(noise=torch.randn((n_chunks,) + shape, generator=g).cuda(),
                    noise_tape=torch.randn((n_chunks, n_steps) + shape, generator=g).cuda())
    if form == "x_T":
        return dict(noise=torch.randn((n_chunks,) + shape, generator=g).cuda())
    if form == "philox":
        return dict(noise_seed=1234, sample_index_base=7)
    return {}


@pytest.fixture(scope="module")
def dip():
    return build()


@pytest.mark.parametrize("case", sorted(CASES))
def test_chain_equals_host_chain(dip, case):
    sampler, skw, guided, text, include_prefix, required, form, use_graph = CASES[case]
    model, diffusion, _ = dip
    B = 3
    n_chunks = -(-required // PRED)
    shape = (B, 263, 1, PRED)
    m = b200mdm.ClassifierFreeSampleModel(model) if guided else model
    if form == "tape" and sampler == "dpm_solver_sample_loop":
        pytest.skip("DPM-Solver++ takes no tape")
    y = make_y(B, n_chunks, guided=guided, text=text)
    kw = dict(skw, model_kwargs={"y": y}, use_graph=use_graph, **noise_kw(form, n_chunks, STEPS, shape))
    if sampler != "dpm_solver_sample_loop":
        kw.setdefault("clip_denoised", False)
    dev, hst = run_both(m, diffusion, sampler, shape, required, include_prefix, **kw)
    assert dev.shape == hst.shape == (B, 263, 1, required)
    assert torch.equal(dev, hst), float((dev - hst).abs().max())
    assert not torch.equal(dev[..., :PRED], dev[..., PRED:2 * PRED])


@pytest.mark.parametrize("what", ["target", "inpaint", "soft_inpaint", "respaced", "longmem", "shape196"])
def test_chain_equals_host_chain_extra(what):
    B, required, pred, ctx, mt, steps, respacing = 3, 30, PRED, CTX, 6, STEPS, None
    if what == "respaced":
        steps, respacing = 20, "5"
    if what == "longmem":
        mt = 200
    if what == "shape196":
        B, required, pred, ctx, steps = 2, 196, 40, 20, 2
    model, diffusion, _ = build(steps=steps, respacing=respacing, target=what == "target", mt=mt, ctx=ctx, pred=pred)
    n_chunks = -(-required // pred)
    shape = (B, 263, 1, pred)
    y = make_y(B, n_chunks, mt=mt, ctx=ctx, pred=pred, text="dynamic" if what == "longmem" else "static")
    if what == "target":
        tg = b200mdm.synthetic_target_inputs(B, seed=5)
        y.update(target_cond=tg["target_cond"].cuda(), target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    if what == "inpaint":
        mask = torch.zeros(shape, dtype=torch.bool)
        mask[..., :3] = True
        y.update(inpainting_mask=mask.cuda(), inpainted_motion=torch.randn(shape).cuda())
    if what == "soft_inpaint":
        y.update(inpainting_weight=torch.rand(shape).cuda(), inpainted_motion=torch.randn(shape).cuda())
    dev, hst = run_both(b200mdm.ClassifierFreeSampleModel(model), diffusion, "ddim_sample_loop", shape, required, True,
                        ctx=ctx, model_kwargs={"y": y}, eta=0.5)
    assert dev.shape == (B, 263, 1, required) and torch.equal(dev, hst)


def test_engine_state_against_fresh_engines():
    model, diffusion, sd = build()
    m = b200mdm.ClassifierFreeSampleModel(model)
    B, shape = 3, (3, 263, 1, PRED)
    y = make_y(B, 4)
    x_T = torch.randn(shape).cuda()
    tape = torch.randn((STEPS,) + shape).cuda()
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=False)

    def chain(mm):
        torch.cuda.manual_seed(3)
        return b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, 30).sample(mm, shape, model_kwargs={"y": y})

    def plain(mm, Bp=B):
        yy = make_y(Bp, 1, seed=8)
        return diffusion.p_sample_loop(mm, (Bp, 263, 1, PRED), noise=x_T[:Bp], noise_tape=tape[:, :Bp], model_kwargs={"y": yy},
                                       clip_denoised=False)
    first = chain(m)
    after_chain = plain(m)
    other = plain(m, 2)                               # another shape, then the chain again
    again = chain(m)
    fresh_model, _, _ = build()
    fm = b200mdm.ClassifierFreeSampleModel(fresh_model)
    assert torch.equal(after_chain, plain(fm))
    assert torch.equal(first, again)
    fresh2, _, _ = build()
    assert torch.equal(again, chain(b200mdm.ClassifierFreeSampleModel(fresh2)))
    assert other.shape[0] == 2


def test_philox_batch_split_equals_whole_batch(dip):
    model, diffusion, _ = dip
    m = b200mdm.ClassifierFreeSampleModel(model)
    B = 4
    y = make_y(B, 4, text="static")
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=True)
    s = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, 30)
    whole = s.sample(m, (B, 263, 1, PRED), model_kwargs={"y": y}, noise_seed=77, clip_denoised=False)
    halves = []
    for lo, hi in ((0, 2), (2, 4)):
        yh = {k: (v[lo:hi] if torch.is_tensor(v) else v) for k, v in y.items()}
        yh["text_embed"] = (y["text_embed"][0][:, lo:hi], y["text_embed"][1][lo:hi])
        halves.append(s.sample(m, (2, 263, 1, PRED), model_kwargs={"y": yh}, noise_seed=77, sample_index_base=lo,
                               clip_denoised=False))
    assert torch.equal(whole, torch.cat(halves))


def test_one_conditioning_upload_and_no_host_sync(dip, monkeypatch):
    model, diffusion, _ = dip
    m = b200mdm.ClassifierFreeSampleModel(model)
    eng = model.engine()
    calls = []
    orig = type(eng).set_cond

    def counting(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(type(eng), "set_cond", counting)
    y = make_y(3, 4, host_mask=True)
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=False)
    s = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, 30)
    s.sample(m, (3, 263, 1, PRED), model_kwargs={"y": y}, clip_denoised=False)        # warm-up: graph capture
    torch.cuda.synchronize()
    assert len(calls) == 1
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = s.sample(m, (3, 263, 1, PRED), model_kwargs={"y": y}, clip_denoised=False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(calls) == 2 and torch.isfinite(out).all()


def test_chain_against_fp32_oracle(dip):
    chain_against_fp32_oracle(*dip, 263)


def chain_against_fp32_oracle(model, diffusion, sd, njoints):
    """A 3-chunk chain (each chunk's prefix handed over on the device) against the fp32 oracle's chunks."""
    m = b200mdm.ClassifierFreeSampleModel(model)
    B, required = 3, 20
    n_chunks = -(-required // PRED)
    shape = (B, njoints, 1, PRED)
    y = make_y(B, n_chunks, njoints=njoints)
    nk = noise_kw("tape", n_chunks, STEPS, shape)
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=False)
    out = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, required).sample(
        m, shape, model_kwargs={"y": y}, clip_denoised=False, **nk)
    W = mo.OracleWeights(sd, L, arch="trans_dec")
    tabs = so.diffusion_tables(so.named_betas("cosine", STEPS))
    enc, tmask = y["text_embed"][0].cpu(), y["text_embed"][1].cpu()
    prefix, pieces = y["prefix"].cpu(), []
    for c in range(n_chunks):
        tape = [nk["noise"][c].cpu()] + list(nk["noise_tape"][c].cpu())
        x = mo.sample_loop_dec(W, tabs, list(range(STEPS)), tape, enc, tmask, prefix, y["scale"].cpu(), y["lengths"].cpu())
        pieces.append(x)
        prefix = x[..., -CTX:]
    ref = torch.cat(pieces, -1)[..., :required]
    assert rel_err(out, ref) < 1e-3


@pytest.mark.parametrize("case", sorted(ga.CASES))
def test_chain_against_the_reference_fixture(golden, case):
    """tests/golden/dip_ar_small.npz: the device chain against the unmodified reference's AutoRegressiveSampler with
    p_sample_loop on the same tape and prompts (oracle/gen_golden_ar_chain.py)."""
    g = golden("dip_ar_small.npz")
    cfg = ga.CASES[case]
    inp = ga.inputs(case)
    over = dict(layers=ga.L, diffusion_steps=ga.STEPS, arch="trans_dec", text_encoder_type="bert", context_len=ga.CTX,
                pred_len=ga.PRED)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=ga.L, cond_dim=C,
                                                                   seed=ga.WEIGHTS_SEED))
    model.to("cuda").eval()
    model.clip_model = ga.TableBert(case, inp["enc"], inp["pad"])
    y = {k: v.cuda() if torch.is_tensor(v) else v for k, v in ga.y_of(case, inp).items()}
    if "text_embed" in y:
        y["text_embed"] = tuple(t.cuda() for t in y["text_embed"])
    calls = []
    eng = model.engine()
    orig = eng.chain_loop_range
    eng.chain_loop_range = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    try:
        out = b200mdm.AutoRegressiveSampler(ga.ar_args(case), diffusion.p_sample_loop, cfg["required"]).sample(
            b200mdm.ClassifierFreeSampleModel(model), (ga.B, 263, 1, cfg["required"]), clip_denoised=False,
            model_kwargs={"y": y}, noise=inp["x_T"].cuda(), noise_tape=inp["eps"].cuda())
    finally:
        del eng.chain_loop_range
    assert calls, "the device chain did not run"
    assert out.shape == g[case + "_sample"].shape
    assert rel_err(out, g[case + "_sample"]) < 1e-3


def test_engine_state_rejections(dip):
    """The C ABI's rejections that need an engine: a non-DiP engine, pred_len / context_len other than the
    conditioning's, a stale DPM-Solver++ table, a chain that was never set up or was ended (by another loop,
    b200mdm_set_cond_dec, b200mdm_set_prefix, or its own last step), steps past the chain, and the conditioning a chain
    consumed."""
    from b200mdm import _lib
    model, diffusion, _ = dip
    m = b200mdm.ClassifierFreeSampleModel(model)
    eng = model.engine()
    lib, h = eng.lib, eng.h
    B, shape = 3, (3, 263, 1, PRED)
    y = make_y(B, 2)
    buf = torch.zeros((2,) + shape, device="cuda")                # x_T of the chain's two chunks
    tape = torch.zeros((2 * STEPS,) + shape, device="cuda")       # an eps row for every step of the chain
    out = torch.zeros(B, 263, 1, 16, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def prepare(dpm=False):
        e = diffusion._prepare(m, shape, {"y": dict(y)}, torch.device("cuda"), 0.0)
        e.set_schedule(diffusion.schedule_rows(0.0), diffusion._timestep_map())     # uploaded again: the DPM table is stale
        if dpm:
            e.set_schedule_dpm(diffusion.schedule_dpm_rows(), key=None)
        return e

    def setup(n=2, pred=PRED, ctx=CTX, crop=16):
        return lib.b200mdm_chain_setup(h, n, pred, ctx, 0, crop, None, None, st)

    def loop(first=0, n=1, mode=_lib.MODE_DDPM, order=0):
        return lib.b200mdm_chain_loop_range(h, mode, order, first, n, buf.data_ptr(), buf[0].numel(), tape.data_ptr(),
                                            tape[0].numel(), out.data_ptr(), 0, 1, st)
    prepare()
    assert setup(pred=PRED + 1) == _lib.EINVAL and setup(ctx=CTX - 1) == _lib.EINVAL
    assert loop() == _lib.ESTATE                                   # never set up
    assert setup() == _lib.OK
    assert loop(first=1) == _lib.ESTATE                            # not where the chain stands
    assert loop(n=2 * STEPS + 1) == _lib.EINVAL                    # past the chain's 2 x STEPS steps
    assert loop(mode=_lib.MODE_DPM, order=2) == _lib.ESTATE        # set_schedule left the DPM-Solver++ table stale
    assert loop(n=STEPS) == _lib.OK and loop(first=STEPS, n=1) == _lib.OK
    # the chain consumed the conditioning: a plain loop needs it set again
    assert lib.b200mdm_sample_loop_range(h, _lib.MODE_DDPM, STEPS - 1, 1, buf.data_ptr(), None, buf.data_ptr(), 0, 0, 1,
                                         st) == _lib.ESTATE
    assert loop(first=STEPS + 1, n=STEPS - 1) == _lib.OK
    assert loop(first=2 * STEPS, n=1) == _lib.ESTATE               # the chain ended with its last step
    for end in ("loop", "cond", "prefix"):
        e = prepare()
        assert setup() == _lib.OK
        if end == "loop":
            e.sample_loop_range(_lib.MODE_DDPM, STEPS - 1, 1, buf[0], None, buf, 0, True)
        elif end == "cond":
            prepare()
        else:
            assert lib.b200mdm_set_prefix(h, y["prefix"].data_ptr(), st) == _lib.OK
        assert loop() == _lib.ESTATE, end
    prepare(dpm=True)
    assert setup() == _lib.OK and loop(mode=_lib.MODE_DPM, order=2, n=2 * STEPS) == _lib.OK
    torch.cuda.synchronize()
    enc_model, _ = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=STEPS),
                                                      SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(enc_model, b200mdm.synthetic_state_dict(num_layers=1, seed=2))
    enc_model.to("cuda").eval()
    enc_eng = enc_model.engine()
    assert enc_eng.lib.b200mdm_chain_setup(enc_eng.h, 2, PRED, CTX, 0, 16, None, None, st) == _lib.EINVAL
    assert enc_eng.lib.b200mdm_chain_loop_range(enc_eng.h, _lib.MODE_DDPM, 0, 0, 1, buf.data_ptr(), 0, buf.data_ptr(), 0,
                                                out.data_ptr(), 0, 1, st) == _lib.EINVAL
