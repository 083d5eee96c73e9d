"""CPU: continuous batching of chains (b200mdm.ContinuousChainSampler, serving.SlotScheduler with n_chunks chunk
boundaries per request) against stand-in engines, and its refusals and argument checks, all raised before any engine
work."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import serving
from b200mdm.serving import SlotScheduler, _Request
from conftest import default_args

N_STEPS, SHAPE = 5, (2, 1, 6)


class FakeChainEngine:
    """Slots as the C ABI keeps them for chains: a slot runs n_steps steps per chunk; it is handed off when it has just
    finished a chunk that is not its last, and read (which frees it) when it has finished its last one.  Every call is
    checked against that contract."""

    def __init__(self, slots):
        self.req = [None] * slots
        self.ran = [0] * slots
        self.chunk = [0] * slots
        self.log = []

    def slot_admit(self, slot, embed, action, scale, length, seed, sample_index):
        assert self.req[slot] is None, "slot %d reused before it was read" % slot
        self.req[slot], self.ran[slot], self.chunk[slot] = sample_index, 0, 0
        self.log.append(("admit", slot, sample_index))

    def slots_run(self, n, use_graph=True):
        assert n > 0
        for b, r in enumerate(self.req):
            if r is not None:
                self.ran[b] = min(N_STEPS, self.ran[b] + n)
        self.log.append(("run", n))

    def slot_handoff(self, slot, r, c):
        assert self.req[slot] == r.sample_index and self.ran[slot] == N_STEPS, "hand-off before the chunk finished"
        assert c == self.chunk[slot] and c + 1 < r.n_chunks
        self.chunk[slot], self.ran[slot] = c + 1, 0
        self.log.append(("handoff", slot, r.sample_index, c))

    def slot_read(self, slot, out):
        assert self.req[slot] is not None and self.ran[slot] == N_STEPS, "slot %d read before it finished" % slot
        out.fill_(float(self.req[slot]))
        self.log.append(("read", slot, self.req[slot], self.chunk[slot]))
        self.req[slot] = None
        return out


def _sched(slots):
    eng = FakeChainEngine(slots)
    return SlotScheduler(eng, slots, N_STEPS, SHAPE, "cpu"), eng


def _submit(s, rid, n_chunks, chain=True):
    out = torch.empty(SHAPE[:-1] + (3 * n_chunks,)) if chain else None
    s.queue.append(_Request(rid, None, 0, 0.0, 3 * n_chunks if chain else 6, 1, rid, n_chunks, out))


def _check_log(log, chunks):
    """Exactly n_chunks x N_STEPS steps per request, a hand-off at each of its chunk boundaries but the last, in chunk
    order, and one read at the last; admissions in submission order."""
    steps, since, seen = 0, {}, {}
    for e in log:
        if e[0] == "run":
            steps += e[1]
        elif e[0] == "admit":
            since[e[2]] = steps
            seen[e[2]] = []
        elif e[0] == "handoff":
            rid, c = e[2], e[3]
            assert steps - since[rid] == (c + 1) * N_STEPS
            seen[rid].append(c)
        else:
            rid = e[2]
            assert steps - since[rid] == chunks[rid] * N_STEPS
            assert seen[rid] == list(range(chunks[rid] - 1))
            seen[rid].append("read")
    assert all(v[-1:] == ["read"] and v.count("read") == 1 for v in seen.values())
    assert sorted(seen) == sorted(chunks)
    admits = [e[2] for e in log if e[0] == "admit"]
    assert admits == sorted(admits)


def test_fixed_trace_hands_off_at_every_chunk_boundary():
    s, eng = _sched(2)
    chunks = {0: 3, 1: 1, 2: 2, 3: 4, 4: 1}
    for rid, n in chunks.items():
        _submit(s, rid, n)
    out = s.step(N_STEPS)                             # 1 finishes; 0 is handed off into its second chunk
    assert [rid for rid, _ in out] == [1]
    assert [e for e in eng.log if e[0] == "handoff"] == [("handoff", 0, 0, 0)]
    out = s.step(N_STEPS)                             # 2 (admitted into 1's slot) runs its first chunk, 0 its second
    assert out == [] and s.active == 2 and s.pending == 2
    out = s.step(N_STEPS)                             # 0 ends its third chunk, 2 its second
    assert [rid for rid, _ in out] == [0, 2]
    for rid, m in out:
        assert m.shape == SHAPE[:-1] + (3 * chunks[rid],) and bool((m == rid).all())
    out = s.drain()
    assert [rid for rid, _ in out] == [4, 3]          # 4 (one chunk) finishes before 3 (four chunks)
    assert s.pending == 0 and s.active == 0
    _check_log(eng.log, chunks)


def test_one_chunk_requests_are_read_as_before():
    s, eng = _sched(2)
    for rid in range(3):
        _submit(s, rid, 1, chain=False)
    out = s.drain()
    assert [rid for rid, _ in out] == [0, 1, 2]
    assert all(m.shape == SHAPE for _, m in out)
    assert not [e for e in eng.log if e[0] == "handoff"]
    _check_log(eng.log, {0: 1, 1: 1, 2: 1})


def test_random_traces_against_the_contract():
    rng = np.random.default_rng(1)
    for trial in range(30):
        slots = int(rng.integers(1, 5))
        s, eng = _sched(slots)
        rid, got, chunks = 0, [], {}
        for _ in range(int(rng.integers(1, 12))):
            for _ in range(int(rng.integers(0, 4))):
                chunks[rid] = int(rng.integers(1, 5))
                _submit(s, rid, chunks[rid])
                rid += 1
            got += [r for r, _ in s.step(int(rng.integers(1, 13)))]
        got += [r for r, _ in s.drain()]
        assert sorted(got) == list(range(rid))
        assert s.pending == 0 and s.active == 0
        _check_log(eng.log, chunks)
        # completion order: a request that was read earlier finished at an earlier (or the same) step
        reads = [e[2] for e in eng.log if e[0] == "read"]
        assert reads == [r for r in got]


# ------------------------------------------------------------------------------------------------ the sampler
PRED, CTX, MT, C = 6, 4, 5, 768


class FakeEngine:
    """Engine.chain_slot_* as the C ABI keeps them: records every call, and checks that each hand-off lands its chunk at
    frame off + c * pred_len and carries chunk c + 1's prompt."""

    def __init__(self):
        self.log = []
        self.state = {}

    def set_schedule(self, *a, **k):
        self.log.append(("schedule",))

    def chain_slots_begin(self, slots, nframes, guided, mode, n_tokens, flags=0):
        self.log.append(("begin", slots, nframes, guided, n_tokens))

    def chain_slot_admit(self, slot, tokens, mask, prefix, scale, length, include_prefix, seed, sample_index):
        assert tokens.shape == (MT, C) and mask.shape == (MT,) and mask.dtype == torch.uint8
        self.state[slot] = dict(g=sample_index, chunk=0, off=CTX if include_prefix else 0, n=-(-length // PRED))
        self.log.append(("admit", slot, sample_index, float(tokens[0, 0])))

    def slots_run(self, n, use_graph=True):
        self.log.append(("run", n))

    def chain_slot_handoff(self, slot, out, tokens=None, mask=None):
        st = self.state[slot]
        self.log.append(("handoff", slot, st["g"], st["chunk"], st["off"] + st["chunk"] * PRED,
                         None if tokens is None else float(tokens[0, 0])))
        st["chunk"] += 1
        if st["chunk"] == st["n"]:
            del self.state[slot]


def _dip(guided=True, **over):
    args = default_args(layers=1, diffusion_steps=N_STEPS, arch="trans_dec", text_encoder_type="bert", pred_len=PRED,
                        context_len=CTX, **over)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), model, diffusion


@pytest.fixture
def fake(monkeypatch):
    eng = FakeEngine()
    calls = []

    real = serving.engine_for

    def engine_for(model):
        calls.append(model)
        if not isinstance(model, (b200mdm.MDM, b200mdm.ClassifierFreeSampleModel)):
            return real(model)                        # TypeError
        return eng, isinstance(model, b200mdm.ClassifierFreeSampleModel)
    monkeypatch.setattr(serving, "engine_for", engine_for)
    return eng, calls


def _prompt(value, n=3):
    tok = torch.full((n, C), float(value))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[-1] = True
    return tok, mask


def test_sampler_hands_each_chunk_its_prompt_and_frame(fake):
    eng, _ = fake
    cfg, model, diffusion = _dip()
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, 2, n_tokens=MT)
    prefix = torch.randn(263, 1, CTX)
    want = {}
    for rid, (length, per_chunk, inc) in enumerate([(17, True, False), (6, False, True), (13, False, False),
                                                    (24, True, True)]):
        n = -(-length // PRED)
        te = [_prompt(10 * rid + c) for c in range(n)] if per_chunk else _prompt(10 * rid)
        cs.submit(text_embed=te, prefix=prefix, length=length, include_prefix=inc, scale=2.0, seed=3)
        want[rid] = [((CTX if inc else 0) + c * PRED, (10 * rid + c + 1) if per_chunk and c + 1 < n else None)
                     for c in range(n)]
    done = cs.drain()
    assert sorted(r for r, _ in done) == [0, 1, 2, 3]
    for rid, motion in done:
        assert motion.shape == (263, 1, [17, 6, 13, 24][rid])
        if rid in (1, 3):                            # include_prefix: the motion starts with the prefix
            assert torch.equal(motion[..., :CTX], prefix[..., :CTX])
    got = {}
    for e in eng.log:
        if e[0] == "admit":
            assert e[3] == 10 * e[2]                  # chunk 0's prompt
        if e[0] == "handoff":
            got.setdefault(e[2], []).append((e[4], e[5]))
    assert got == want
    assert [e for e in eng.log if e[0] == "begin"] == [("begin", 2, PRED, True, MT)]


def test_refusals_before_engine_work(fake):
    _, calls = fake
    cfg, model, diffusion = _dip()
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=MT, sampler="plms")
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=MT, sampler="dpm_solver")
    with pytest.raises(ValueError):
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=MT, eta=0.5)
    with pytest.raises(ValueError):
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=513)
    with pytest.raises(ValueError):
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=0)
    with pytest.raises(ValueError):                   # a DiP slot is one pred_len chunk
        b200mdm.ContinuousChainSampler(diffusion, cfg, 4, n_tokens=MT, nframes=PRED + 1)
    enc, ediff = b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4),
                                                    SimpleNamespace(dataset=SimpleNamespace()))
    with pytest.raises(ValueError):                   # no BERT memory: ContinuousSampler's model
        b200mdm.ContinuousChainSampler(ediff, b200mdm.ClassifierFreeSampleModel(enc), 4, n_tokens=MT)
    bert, bdiff = b200mdm.create_model_and_diffusion(
        default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert"),
        SimpleNamespace(dataset=SimpleNamespace()))
    with pytest.raises(ValueError):                   # the plain BERT decoder needs its slot's frame count
        b200mdm.ContinuousChainSampler(bdiff, bert, 4, n_tokens=MT)
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousChainSampler(bdiff, b200mdm.HandshakeSampleModel(bert, 2), 4, n_tokens=MT, nframes=20)
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousChainSampler(bdiff, b200mdm.MultiPromptSampleModel(bert), 4, n_tokens=MT, nframes=20)
    assert calls == []
    with pytest.raises(TypeError):                    # a model this package does not drive
        b200mdm.ContinuousChainSampler(diffusion, torch.nn.Linear(2, 2), 4, n_tokens=MT)


def test_submit_checks_before_engine_work(fake):
    eng, _ = fake
    cfg, model, diffusion = _dip()
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, 2, n_tokens=MT)
    prefix = torch.randn(263, 1, CTX)
    n0 = len(eng.log)
    bad = [
        dict(text_embed=_prompt(1, n=MT + 1), prefix=prefix, scale=1.0),                  # more tokens than n_tokens
        dict(text_embed=_prompt(1), scale=1.0),                                           # DiP without a prefix
        dict(text_embed=_prompt(1), prefix=torch.randn(263, 1, CTX + 1), scale=1.0),      # prefix of the wrong shape
        dict(text_embed=_prompt(1), prefix=torch.randn(251, 1, CTX), scale=1.0),
        dict(text_embed=[_prompt(1), _prompt(2)], prefix=prefix, length=3 * PRED, scale=1.0),   # 2 prompts, 3 chunks
        dict(text_embed=_prompt(1), prefix=prefix, length=0, scale=1.0),                  # length below 1
        dict(text_embed=_prompt(1), prefix=prefix),                                       # guided without a scale
        dict(prefix=prefix, scale=1.0),                                                   # no prompt
        dict(text_embed=(torch.zeros(3, C), torch.zeros(4)), prefix=prefix, scale=1.0),   # tokens / mask disagree
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            cs.submit(seed=1, **kw)
    assert cs.pending == 0 and len(eng.log) == n0
    assert cs.submit(text_embed=[_prompt(1), _prompt(2)], prefix=prefix[None], length=2 * PRED, scale=1.0, seed=1) == 0

    plain, _, pdiff = _dip(guided=False)
    cp = b200mdm.ContinuousChainSampler(pdiff, plain, 2, n_tokens=MT, sampler="ddim", eta=0.5)
    with pytest.raises(ValueError):
        cp.submit(text_embed=_prompt(1), prefix=prefix, scale=1.0, seed=1)               # scale without guidance
    bert, bdiff = b200mdm.create_model_and_diffusion(
        default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="bert"),
        SimpleNamespace(dataset=SimpleNamespace()))
    cb = b200mdm.ContinuousChainSampler(bdiff, bert, 2, n_tokens=MT, nframes=20)
    n0 = len(eng.log)
    for kw in (dict(text_embed=_prompt(1), prefix=prefix),                              # no prefix on this model
               dict(text_embed=_prompt(1), include_prefix=True),
               dict(text_embed=_prompt(1), length=21),                                  # one chunk of <= 20 frames
               dict(text_embed=[_prompt(1), _prompt(2)], length=20)):                   # one chunk, one prompt
        with pytest.raises(ValueError):
            cb.submit(seed=1, **kw)
    assert cb.pending == 0 and len(eng.log) == n0
    assert cb.submit(text_embed=_prompt(1), length=7, seed=1) == 0


def test_continuous_sampler_still_refuses_dip():
    cfg, model, diffusion = _dip()
    with pytest.raises(NotImplementedError, match="ContinuousChainSampler"):
        b200mdm.ContinuousSampler(diffusion, cfg, 4, PRED)
