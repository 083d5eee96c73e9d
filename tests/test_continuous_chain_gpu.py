"""GPU: continuous batching of DiP chains and of the plain BERT decoder (b200mdm.ContinuousChainSampler,
b200mdm_chain_slots_*).

The main property is request identity: a DiP request with (seed s, sample index g) admitted into slot b, at any step and
whatever runs in the other slots, is bitwise row b of AutoRegressiveSampler(p_sample_loop / ddim_sample_loop) with
noise_seed = s and sample_index_base = g - b at the same slots, pred_len, context_len and memory width, with the
request's prefix, prompt(s) and scale at row b.  The device chain itself is tied to the unmodified reference's
AutoRegressiveSampler by tests/test_ar_chain_gpu.py (tests/golden/dip_ar_small.npz)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from conftest import default_args

pytestmark = pytest.mark.gpu
B, L, CTX, PRED, STEPS, C = 4, 2, 8, 12, 5, 768


class FakeBert:
    """A deterministic stand-in for the DistilBERT wrapper (as in tests/test_ar_chain_gpu.py): features seeded by the
    text, `mt` tokens, the first 1 + len(text) % mt present."""

    def __init__(self, mt):
        self.mt = mt

    def __call__(self, texts):
        enc = torch.stack([torch.randn(self.mt, C, generator=torch.Generator().manual_seed(sum(map(ord, t)) + 7))
                           for t in texts]).cuda()
        present = torch.zeros(len(texts), self.mt, dtype=torch.bool)
        for b, t in enumerate(texts):
            present[b, :1 + len(t) % self.mt] = True
        return enc, present.cuda()


def _build(mt, ctx=CTX, pred=PRED, seed=21):
    over = dict(layers=L, diffusion_steps=STEPS, arch="trans_dec", text_encoder_type="bert", context_len=ctx, pred_len=pred)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=C, seed=seed))
    model.to("cuda").eval()
    model.clip_model = FakeBert(mt)
    return model, diffusion


class Recorder:
    """Forwards to the scheduler's engine and records which slot each request (by sample index) was admitted into."""

    def __init__(self, eng):
        self.eng, self.slot_of = eng, {}

    def slot_admit(self, slot, embed, action, scale, length, seed, sample_index):
        self.slot_of[sample_index] = slot
        self.eng.slot_admit(slot, embed, action, scale, length, seed, sample_index)

    def slots_run(self, n, use_graph=True):
        self.eng.slots_run(n, use_graph)

    def slot_handoff(self, slot, r, c):
        self.eng.slot_handoff(slot, r, c)

    def slot_read(self, slot, out):
        return self.eng.slot_read(slot, out)


def _dip_request(rng, i, mt, guided):
    """Request i of a trace: lengths over 1 .. 4 chunks (not all multiples of PRED), static or per-chunk prompts, as text
    (FakeBert) or as a (tokens, mask) pair shorter than the memory width, include_prefix on or off."""
    length = [2 * PRED + 3, PRED, 1, 4 * PRED, 3 * PRED - 1, 5, PRED + 1, 2 * PRED, 3 * PRED + 7][i % 9]
    n_chunks = -(-length // PRED)
    r = dict(length=length, include_prefix=bool(i % 2), seed=int(rng.integers(1, 2 ** 40)),
             prefix=torch.from_numpy(rng.standard_normal((263, 1, CTX)).astype(np.float32)))
    kind = ["text", "chunks", "embed"][i % 3]
    if kind == "text":
        r["text"] = "request %d" % i + "." * int(rng.integers(0, 9))
    elif kind == "chunks":
        r["text"] = ["request %d, chunk %d" % (i, c) + "," * int(rng.integers(0, 9)) for c in range(n_chunks)]
    else:
        n = int(rng.integers(1, mt))                  # fewer tokens than the width
        r["text_embed"] = (torch.from_numpy(rng.standard_normal((n, C)).astype(np.float32)),
                           torch.from_numpy(rng.random(n) < 0.3) & torch.tensor([False] + [True] * (n - 1)))
    if guided:
        r["scale"] = float(rng.uniform(0.5, 7.5))
    return r


def _dip_reference(model, diffusion, req, slot, g, guided, sampler, eta, mt, use_graph):
    """Row `slot` of the uniform device chain that the request must reproduce; the other rows run other prompts."""
    n_chunks = -(-req["length"] // PRED)
    others = torch.randn(B, 263, 1, CTX, generator=torch.Generator().manual_seed(5))
    prefix = others.clone()
    prefix[slot] = req["prefix"]
    y = dict(prefix=prefix.cuda(), mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"))
    text = req.get("text")
    if isinstance(text, list):
        y["text"] = [["other %d chunk %d" % (b, c) for c in range(n_chunks)] for b in range(B)]
        y["text"][slot] = text
        y["text_embed"] = (torch.zeros(mt, B, n_chunks, C, device="cuda"), torch.zeros(B, n_chunks, mt, dtype=torch.bool,
                                                                                         device="cuda"))
    elif text is not None:
        y["text"] = ["other %d" % b for b in range(B)]
        y["text"][slot] = text
    else:
        enc, pad = model.clip_model(["other %d" % b for b in range(B)])
        enc, pad = enc.permute(1, 0, 2).contiguous(), ~pad
        tok, m = req["text_embed"]
        enc[:, slot] = 0.0
        enc[:tok.shape[0], slot] = tok.cuda()
        pad[slot] = True
        pad[slot, :tok.shape[0]] = m.cuda()
        y["text_embed"] = (enc, pad)
    if guided:
        y["scale"] = torch.full((B,), 1.0, device="cuda")
        y["scale"][slot] = req["scale"]
    cfg = b200mdm.ClassifierFreeSampleModel(model) if guided else model
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=req["include_prefix"])
    fn, kw = (diffusion.p_sample_loop, {}) if sampler == "ddpm" else (diffusion.ddim_sample_loop, {"eta": eta})
    out = b200mdm.AutoRegressiveSampler(args, fn, required_frames=req["length"]).sample(
        cfg, (B, 263, 1, PRED), model_kwargs={"y": y}, clip_denoised=False, noise_seed=req["seed"],
        sample_index_base=g - slot, use_graph=use_graph, **kw)
    return out[slot]


def _dip_trace(guided=True, sampler="ddpm", eta=0.0, use_graph=True, mt=8, n_req=9, seed=0):
    model, diffusion = _build(mt)
    cfg = b200mdm.ClassifierFreeSampleModel(model) if guided else model
    rng = np.random.default_rng(seed)
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, B, n_tokens=mt, sampler=sampler, eta=eta, use_graph=use_graph)
    rec = Recorder(cs.scheduler.engine)
    cs.scheduler.engine = rec
    reqs = {}
    count = [0]

    def submit(k):
        for _ in range(k):
            r = _dip_request(rng, count[0], mt, guided)
            count[0] += 1
            rid = cs.submit(**r, sample_index=int(rng.integers(B, 10 ** 6)))
            reqs[rid] = (r, cs.scheduler.queue[-1].sample_index)

    done = []
    submit(3)
    done += cs.step(2)
    submit(4)
    done += cs.step(STEPS + 3)
    submit(n_req - 7)
    done += cs.step(1)
    done += cs.drain()
    assert sorted(rid for rid, _ in done) == list(range(n_req))
    assert cs.pending == 0 and cs.active == 0
    for rid, motion in done:
        r, g = reqs[rid]
        ref = _dip_reference(model, diffusion, r, rec.slot_of[g], g, guided, sampler, eta, mt, use_graph)
        assert motion.shape == ref.shape == (263, 1, r["length"])
        assert torch.equal(motion, ref), (guided, sampler, eta, rid, float((motion - ref).abs().max()))


def test_request_identity_dip_guided():
    _dip_trace(True)


def test_request_identity_dip_unguided():
    _dip_trace(False, seed=1)


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_request_identity_dip_ddim(eta):
    _dip_trace(True, sampler="ddim", eta=eta, seed=2)


def test_request_identity_dip_without_graph():
    _dip_trace(True, use_graph=False, n_req=7, seed=3)


def test_request_identity_dip_key_blocked_memory():
    _dip_trace(True, mt=80, n_req=7, seed=4)               # a width above 64: the key-blocked cross-attention


def test_request_identity_bert_decoder():
    """The plain BERT decoder (context_len 0): a request is one chunk whose length masks its frames, row b of
    p_sample_loop with per-row lengths."""
    T, mt = 24, 8
    model, diffusion = _build(mt, ctx=0, pred=0)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    rng = np.random.default_rng(6)
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, B, n_tokens=mt, nframes=T)
    rec = Recorder(cs.scheduler.engine)
    cs.scheduler.engine = rec
    reqs = {}

    def submit(k):
        for _ in range(k):
            n = int(rng.integers(1, mt + 1))
            r = dict(length=int(rng.integers(1, T + 1)), scale=float(rng.uniform(0.5, 7.5)), seed=int(rng.integers(1, 2 ** 40)),
                     text_embed=(torch.from_numpy(rng.standard_normal((n, C)).astype(np.float32)),
                                 torch.tensor([False] + [bool(v) for v in rng.random(n - 1) < 0.3])))
            rid = cs.submit(**r, sample_index=int(rng.integers(B, 10 ** 6)))
            reqs[rid] = (r, cs.scheduler.queue[-1].sample_index)
    done = []
    submit(3)
    done += cs.step(2)
    submit(4)
    done += cs.step(3)
    submit(1)
    done += cs.drain()
    assert sorted(rid for rid, _ in done) == list(range(8))
    for rid, motion in done:
        r, g = reqs[rid]
        slot = rec.slot_of[g]
        enc, pad = model.clip_model(["other %d" % b for b in range(B)])
        enc, pad = enc.permute(1, 0, 2).contiguous(), ~pad
        tok, m = r["text_embed"]
        enc[:, slot] = 0.0
        enc[:tok.shape[0], slot] = tok.cuda()
        pad[slot] = True
        pad[slot, :tok.shape[0]] = m.cuda()
        lengths = torch.full((B,), T, dtype=torch.int64, device="cuda")
        lengths[slot] = r["length"]
        scale = torch.full((B,), 2.0, device="cuda")
        scale[slot] = r["scale"]
        y = dict(text_embed=(enc, pad), lengths=lengths, scale=scale,
                 mask=(torch.arange(T, device="cuda")[None, :] < lengths[:, None]).reshape(B, 1, 1, T))
        ref = diffusion.p_sample_loop(cfg, (B, 263, 1, T), model_kwargs={"y": y}, clip_denoised=False,
                                      noise_seed=r["seed"], sample_index_base=g - slot)[slot, ..., :r["length"]]
        assert motion.shape == ref.shape and torch.equal(motion, ref), rid


def test_slot_graph_launches_as_many_kernels_as_the_uniform_graph():
    model, diffusion = _build(8)
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    eng = model.engine()
    enc, pad, prefix = b200mdm.synthetic_dip_inputs(B, 8, CTX)
    y = dict(prefix=prefix.cuda(), text_embed=(enc.cuda(), pad.cuda()), scale=torch.full((B,), 2.5, device="cuda"),
             mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"))
    diffusion.p_sample_loop(cfg, (B, 263, 1, PRED), model_kwargs={"y": y}, noise_seed=1)   # capture the uniform graph
    x = eng.philox_normal((B, 263, 1, PRED), 1, 0, -1, "cuda")
    out = torch.empty_like(x)
    eng.launch_count(reset=True)
    eng.sample_loop_range(_lib.MODE_DDPM, STEPS - 1, STEPS, x, out, None, 0, True)
    uniform = eng.launch_count(reset=True) - 1                       # the step_set kernel ahead of the steps
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, B, n_tokens=8)
    cs.submit(text="a request", prefix=prefix[0], length=2 * PRED, scale=2.5, seed=1)
    cs.step(1)                                                       # admission, and the graph's capture
    eng.launch_count(reset=True)
    cs.step(STEPS - 2)                                               # no chunk boundary in these steps
    slot = eng.launch_count(reset=True)
    torch.cuda.synchronize()
    assert slot * STEPS == uniform * (STEPS - 2), (slot, uniform)


def test_admission_and_handoff_launch_counts():
    """The counts include/b200mdm.h states: admission 5 (4 without a prefix), hand-off 4 (6 with a new prompt), the
    last hand-off 1; and a hand-off away from a chunk boundary is refused."""
    mt = 8
    model, diffusion = _build(mt)
    eng = model.engine()
    cs = b200mdm.ContinuousChainSampler(diffusion, b200mdm.ClassifierFreeSampleModel(model), B, n_tokens=mt)
    tok = torch.randn(mt, C, device="cuda")
    mask = torch.zeros(mt, dtype=torch.uint8, device="cuda")
    prefix = torch.randn(263, CTX, device="cuda")
    out = torch.empty(263, 3 * PRED, device="cuda")
    eng.launch_count(reset=True)
    eng.chain_slot_admit(1, tok, mask, prefix, 2.0, 3 * PRED, True, 5, 9)
    assert eng.launch_count(reset=True) == 5
    eng.slots_run(STEPS - 1)
    with pytest.raises(RuntimeError):                                # one step of the chunk is still to run
        eng.chain_slot_handoff(1, out)
    eng.slots_run(1)
    eng.launch_count(reset=True)
    eng.chain_slot_handoff(1, out)
    assert eng.launch_count(reset=True) == 4
    eng.slots_run(STEPS)
    eng.launch_count(reset=True)
    eng.chain_slot_handoff(1, out, tok, mask)
    assert eng.launch_count(reset=True) == 6
    eng.slots_run(STEPS)
    eng.launch_count(reset=True)
    eng.chain_slot_handoff(1, out)
    assert eng.launch_count(reset=True) == 1
    with pytest.raises(RuntimeError):                                # the slot is free
        eng.chain_slot_handoff(1, out)
    bert, bdiff = _build(mt, ctx=0, pred=0)
    beng = bert.engine()
    b200mdm.ContinuousChainSampler(bdiff, bert, B, n_tokens=mt, nframes=24)
    beng.launch_count(reset=True)
    beng.chain_slot_admit(0, tok, mask, None, 0.0, 20, False, 5, 9)
    assert beng.launch_count(reset=True) == 4
    torch.cuda.synchronize()


@pytest.mark.parametrize("use_graph", [True, False])
def test_engine_after_a_slot_session_equals_a_fresh_engine(use_graph):
    mt = 8
    model, diffusion = _build(mt, seed=5)
    model2, _ = _build(mt, seed=5)
    cs = b200mdm.ContinuousChainSampler(diffusion, b200mdm.ClassifierFreeSampleModel(model), B, n_tokens=mt,
                                        sampler="ddim", eta=0.5)
    rng = np.random.default_rng(4)
    for i in range(6):
        cs.submit(**_dip_request(rng, i, mt, True))
    cs.step(STEPS + 2)                                               # leave the session mid-flight, mid-chain
    enc, pad, prefix = b200mdm.synthetic_dip_inputs(B, mt, CTX, seed=9)

    def y():
        return dict(prefix=prefix.cuda(), text_embed=(enc.cuda(), pad.cuda()), scale=torch.tensor([2.5, 1.0, 7.5, 0.0]).cuda(),
                    mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"),
                    lengths=torch.tensor([PRED, 7, 3, 10]).cuda())
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=True)
    outs = []
    for m in (model, model2):
        cfg = b200mdm.ClassifierFreeSampleModel(m)
        chain = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, 30).sample(
            cfg, (B, 263, 1, PRED), model_kwargs={"y": y()}, noise_seed=11, use_graph=use_graph)
        plain = diffusion.p_sample_loop(cfg, (B, 263, 1, PRED), model_kwargs={"y": y()}, noise_seed=11,
                                        use_graph=use_graph)
        outs.append((chain, plain))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    with pytest.raises(RuntimeError):                                # the loops ended the slot session
        cs.step(1)


def test_engine_refusals():
    """b200mdm_slots_begin still refuses BERT-memory engines, the chain entry points refuse other engines, and the
    per-sample step still refuses DiP."""
    model, diffusion = _build(8)
    eng = model.engine()
    eng.set_schedule(diffusion.schedule_rows(0.0), diffusion._timestep_map())
    with pytest.raises(RuntimeError, match="BERT"):
        eng.slots_begin(B, PRED, True, _lib.MODE_DDPM)
    with pytest.raises(RuntimeError):
        eng.chain_slots_begin(B, PRED, True, _lib.MODE_DDPM, 513)
    with pytest.raises(RuntimeError):
        eng.chain_slots_begin(B, PRED, True, _lib.MODE_DPM, 8)
    enc_model, ediff = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=STEPS),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(enc_model, b200mdm.synthetic_state_dict(num_layers=1, seed=2))
    enc_model.to("cuda").eval()
    eeng = enc_model.engine()
    eeng.set_schedule(ediff.schedule_rows(0.0), ediff._timestep_map())
    with pytest.raises(RuntimeError):
        eeng.chain_slots_begin(B, 24, True, _lib.MODE_DDPM, 8)
    enc, pad, prefix = b200mdm.synthetic_dip_inputs(B, 8, CTX)
    y = dict(prefix=prefix.cuda(), text_embed=(enc.cuda(), pad.cuda()), mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool).cuda())
    with pytest.raises(NotImplementedError):                         # mixed t on DiP
        diffusion.p_sample(model, torch.zeros(B, 263, 1, PRED, device="cuda"), torch.tensor([0, 1, 2, 3], device="cuda"),
                           model_kwargs={"y": y})
