"""GPU: continuous batching (b200mdm.ContinuousSampler, b200mdm_slots_*) and p_sample / ddim_sample at a schedule index
per sample (b200mdm_sample_step_at).

The main property is request identity: a request with (seed s, sample index g) admitted into slot b, at any step and
whatever runs in the other slots, is bitwise row b of a uniform Philox loop with noise_seed = s, sample_index_base =
g - b, the same batch and frame count, and the request's conditioning at row b."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from conftest import default_args

pytestmark = pytest.mark.gpu
B, T, STEPS = 4, 24, 5


def _build(kind, guided, seed=1, steps=STEPS):
    over = {}
    sd_kw = {}
    if kind == "a2m":
        over = dict(dataset="humanact12", cond_mask_prob=0.0)
        sd_kw = dict(input_feats=150, cond_mode="action", num_actions=12)
    elif kind == "clipdec":
        over = dict(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
        sd_kw = dict(arch="trans_dec", cond_dim=512)
    args = default_args(layers=2, diffusion_steps=steps, **over)
    data = SimpleNamespace(dataset=SimpleNamespace(**({"num_actions": 12} if kind == "a2m" else {})))
    model, diffusion = b200mdm.create_model_and_diffusion(args, data)
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=2, seed=seed, **sd_kw))
    model.to("cuda").eval()
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), model, diffusion


class Recorder:
    """Forwards to the engine and records which slot each request (by sample index) was admitted into."""

    def __init__(self, eng):
        self.eng, self.slot_of = eng, {}

    def slot_admit(self, slot, embed, action, scale, length, seed, sample_index):
        self.slot_of[sample_index] = slot
        self.eng.slot_admit(slot, embed, action, scale, length, seed, sample_index)

    def slots_run(self, n, use_graph=True):
        self.eng.slots_run(n, use_graph)

    def slot_read(self, slot, out):
        return self.eng.slot_read(slot, out)


def _request(kind, rng):
    r = dict(length=int(rng.integers(3, T + 1)), seed=int(rng.integers(1, 2 ** 40)))
    if kind == "a2m":
        r["action"] = int(rng.integers(0, 12))
    else:
        r["text_embed"] = torch.from_numpy(rng.standard_normal(512).astype(np.float32))
    return r


def _uniform(kind, cfg, model, diffusion, req, slot, g, guided, sampler, eta):
    """Row `slot` of the uniform Philox loop that the request must reproduce."""
    lengths = torch.full((B,), req["length"], dtype=torch.int64, device="cuda")
    mask = (torch.arange(T, device="cuda")[None, :] < lengths[:, None]).reshape(B, 1, 1, T)
    y = dict(lengths=lengths, mask=mask)
    if kind == "a2m":
        y["action"] = torch.full((B, 1), req["action"], dtype=torch.int64, device="cuda")
    else:
        y["text_embed"] = req["text_embed"].to("cuda").reshape(1, 1, -1).expand(1, B, -1).contiguous()
    if guided:
        y["scale"] = torch.full((B,), req["scale"], device="cuda")
    shape = (B, model.njoints, model.nfeats, T)
    kw = dict(clip_denoised=False, model_kwargs={"y": y}, noise_seed=req["seed"], sample_index_base=g - slot)
    if sampler == "ddpm":
        out = diffusion.p_sample_loop(cfg, shape, **kw)
    else:
        out = diffusion.ddim_sample_loop(cfg, shape, eta=eta, **kw)
    return out[slot, ..., :req["length"]]


def _trace(kind, guided, sampler="ddpm", eta=0.0, use_graph=True, n_req=9, seed=0):
    """A trace of more requests than slots, some submitted while others run; every motion against its uniform loop."""
    cfg, model, diffusion = _build(kind, guided)
    rng = np.random.default_rng(seed)
    cs = b200mdm.ContinuousSampler(diffusion, cfg, B, T, sampler=sampler, eta=eta, use_graph=use_graph)
    rec = Recorder(cs.scheduler.engine)
    cs.scheduler.engine = rec
    reqs = {}

    def submit(k):
        for _ in range(k):
            r = _request(kind, rng)
            if guided:
                r["scale"] = float(rng.uniform(0.5, 7.5))
            rid = cs.submit(**r, sample_index=int(rng.integers(B, 10 ** 6)))
            reqs[rid] = (r, cs.scheduler.queue[-1].sample_index)

    done = []
    submit(3)
    done += cs.step(2)
    submit(4)
    done += cs.step(3)
    submit(n_req - 7)
    done += cs.step(1)
    done += cs.drain()
    assert sorted(rid for rid, _ in done) == list(range(n_req))
    assert cs.pending == 0 and cs.active == 0
    for rid, motion in done:
        r, g = reqs[rid]
        ref = _uniform(kind, cfg, model, diffusion, r, rec.slot_of[g], g, guided, sampler, eta)
        assert motion.shape == ref.shape
        assert torch.equal(motion, ref), (kind, guided, sampler, eta, rid)


@pytest.mark.parametrize("guided", [True, False])
def test_request_identity_text(guided):
    _trace("enc", guided)


def test_request_identity_a2m():
    _trace("a2m", False)


def test_request_identity_clip_decoder():
    _trace("clipdec", True)


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_request_identity_ddim(eta):
    _trace("enc", True, sampler="ddim", eta=eta)


def test_request_identity_without_graph():
    _trace("enc", True, use_graph=False, n_req=7)


def test_slot_graph_launches_as_many_kernels_as_the_uniform_graph():
    cfg, model, diffusion = _build("enc", True)
    eng = model.engine()
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=STEPS, seed=3)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=torch.full((B,), 2.5, device="cuda"))
    diffusion.p_sample_loop(cfg, (B, 263, 1, T), model_kwargs={"y": y}, noise_seed=1)   # capture the uniform graph
    x = eng.philox_normal((B, 263, 1, T), 1, 0, -1, "cuda")
    out = torch.empty_like(x)
    eng.launch_count(reset=True)
    eng.sample_loop_range(_lib.MODE_DDPM, STEPS - 1, STEPS, x, out, None, 0, True)
    uniform = eng.launch_count(reset=True) - 1                       # the step_set kernel ahead of the steps
    cs = b200mdm.ContinuousSampler(diffusion, cfg, B, T)
    cs.submit(text_embed=inp["text_embed"][0, 0], scale=2.5, seed=1)
    cs.step(1)                                                       # admission, and the graph's capture
    eng.launch_count(reset=True)
    cs.step(STEPS - 1)
    slot = eng.launch_count(reset=True)
    torch.cuda.synchronize()
    assert slot * STEPS == uniform * (STEPS - 1), (slot, uniform)


def test_engine_after_a_slot_session_equals_a_fresh_engine():
    cfg, model, diffusion = _build("enc", True, seed=5)
    cfg2, model2, _ = _build("enc", True, seed=5)
    cs = b200mdm.ContinuousSampler(diffusion, cfg, B, T, sampler="ddim", eta=0.5)
    rng = np.random.default_rng(4)
    for _ in range(6):
        cs.submit(**_request("enc", rng), scale=3.0)
    cs.step(7)                                                       # leave the session mid-flight
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=STEPS, seed=9, lengths=[24, 17, 5, 12],
                                   scale=torch.tensor([2.5, 1.0, 7.5, 0.0]))
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    for use_graph in (True, False):
        a = diffusion.p_sample_loop(cfg, (B, 263, 1, T), model_kwargs={"y": dict(y)}, noise_seed=11, use_graph=use_graph)
        b = diffusion.p_sample_loop(cfg2, (B, 263, 1, T), model_kwargs={"y": dict(y)}, noise_seed=11, use_graph=use_graph)
        assert torch.equal(a, b)
    with pytest.raises(RuntimeError):                                # the loop ended the slot session
        cs.step(1)


@pytest.mark.parametrize("sampler,eta", [("ddpm", 0.0), ("ddim", 0.0), ("ddim", 0.5)])
@pytest.mark.parametrize("clip", [False, True])
def test_mixed_t_rows_equal_uniform_steps(sampler, eta, clip):
    cfg, model, diffusion = _build("enc", True, steps=8)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=8, seed=21, lengths=[24, 17, 5, 12],
                                   scale=torch.tensor([2.5, 1.0, 7.5, 0.0]))
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 263, 1, T, generator=g).cuda()
    eps = torch.randn(B, 263, 1, T, generator=g).cuda()
    t = torch.tensor([7, 0, 3, 5], device="cuda")
    step = diffusion.p_sample if sampler == "ddpm" else (
        lambda *a, **k: diffusion.ddim_sample(*a, eta=eta, **k))
    mixed = step(cfg, x, t, clip_denoised=clip, model_kwargs={"y": dict(y)}, noise=eps)
    for b in range(B):
        uni = step(cfg, x, torch.full_like(t, int(t[b])), clip_denoised=clip, model_kwargs={"y": dict(y)}, noise=eps)
        for k in ("sample", "pred_xstart"):
            assert torch.equal(mixed[k][b], uni[k][b]), (b, k)


def test_mixed_t_refusals():
    cfg, model, diffusion = _build("enc", True)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=STEPS, seed=2)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=torch.full((B,), 2.5, device="cuda"))
    x = torch.zeros(B, 263, 1, T, device="cuda")
    t = torch.tensor([0, 1, 2, 3], device="cuda")
    with pytest.raises(NotImplementedError):
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": y}, const_noise=True)
    with pytest.raises(NotImplementedError):
        yi = dict(y, inpainting_mask=torch.zeros_like(x, dtype=torch.bool), inpainted_motion=x)
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": yi})
    with pytest.raises(AssertionError):                              # p_mean_variance keeps one index per batch
        diffusion.p_mean_variance(cfg, x, t, model_kwargs={"y": y})


def test_mixed_t_against_the_reference_golden():
    from oracle import gen_golden_mixed_t as gm
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "mixed_t_small.npz"))
    cfg, model, diffusion = _build("enc", True, steps=gm.STEPS)
    inp, x, eps = gm.inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    t = torch.tensor(gm.TS, device="cuda")
    for name, eta in (("ddpm", None), ("ddim_eta0", 0.0), ("ddim_eta0.5", 0.5)):
        kw = dict(clip_denoised=False, model_kwargs={"y": dict(y)}, noise=eps.cuda())
        o = diffusion.p_sample(cfg, x.cuda(), t, **kw) if eta is None else diffusion.ddim_sample(cfg, x.cuda(), t, eta=eta, **kw)
        for k in ("sample", "pred_xstart"):
            ref = torch.from_numpy(g["%s_%s" % (name, k)]).double()
            err = float((o[k].cpu().double() - ref).norm() / ref.norm())
            assert err < 1e-3, (name, k, err)
