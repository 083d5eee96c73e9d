"""CPU: the continuous-batching scheduler (serving.SlotScheduler) against a stand-in engine, and the refusals of
ContinuousSampler and of p_sample / ddim_sample at a schedule index per sample, all raised before any engine work."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm.serving import SlotScheduler, _Request
from conftest import default_args

N_STEPS, SHAPE = 5, (2, 1, 6)


class FakeEngine:
    """Slots as the C ABI keeps them: a slot runs n_steps steps after its admission, then holds its sample until read.
    Every call is checked against that contract."""

    def __init__(self, slots):
        self.req = [None] * slots
        self.ran = [0] * slots
        self.log = []

    def slot_admit(self, slot, embed, action, scale, length, seed, sample_index):
        assert self.req[slot] is None, "slot %d reused before it was read" % slot
        self.req[slot] = sample_index
        self.ran[slot] = 0
        self.log.append(("admit", slot, sample_index))

    def slots_run(self, n, use_graph=True):
        assert n > 0
        for b, r in enumerate(self.req):
            if r is not None:
                self.ran[b] = min(N_STEPS, self.ran[b] + n)
        self.log.append(("run", n))

    def slot_read(self, slot, out):
        assert self.req[slot] is not None and self.ran[slot] == N_STEPS, "slot %d read before it finished" % slot
        out.fill_(float(self.req[slot]))
        self.req[slot] = None
        self.log.append(("read", slot))
        return out


def _sched(slots):
    eng = FakeEngine(slots)
    return SlotScheduler(eng, slots, N_STEPS, SHAPE, "cpu"), eng


def _submit(s, rid, length=6):
    s.queue.append(_Request(rid, None, 0, 0.0, length, 1, rid))


def test_fifo_admission_and_exact_step_count():
    s, eng = _sched(2)
    for rid in range(5):
        _submit(s, rid, length=rid + 1)
    assert s.pending == 5 and s.active == 0
    out = s.step(1)
    assert out == [] and s.pending == 3 and s.active == 2
    assert [e for e in eng.log if e[0] == "admit"] == [("admit", 0, 0), ("admit", 1, 1)]
    out = s.step(4)                                   # requests 0 and 1 finish at step 5, 2 and 3 take their slots
    assert [rid for rid, _ in out] == [0, 1]
    for rid, m in out:
        assert m.shape == SHAPE[:-1] + (rid + 1,) and bool((m == rid).all())
    out = s.step(3)
    assert out == [] and s.active == 2 and s.pending == 1
    out = s.drain()
    assert [rid for rid, _ in out] == [2, 3, 4]
    assert s.pending == 0 and s.active == 0
    # every request ran exactly N_STEPS steps between its admission and its read
    steps, since = 0, {}
    for e in eng.log:
        if e[0] == "run":
            steps += e[1]
        elif e[0] == "admit":
            since[e[1]] = steps
        else:
            assert steps - since[e[1]] == N_STEPS


def test_submissions_between_steps_keep_fifo_and_completion_order():
    s, eng = _sched(3)
    _submit(s, 0)
    s.step(2)
    _submit(s, 1)
    _submit(s, 2)
    _submit(s, 3)
    _submit(s, 4)
    out = s.step(3)                                   # 0 finishes after 3 more steps; 1, 2 are 3 steps in
    assert [rid for rid, _ in out] == [0]
    out = s.step(2)                                   # 1 and 2 finish together: by id; 3 went into 0's slot
    assert [rid for rid, _ in out] == [1, 2]
    admits = [e[2] for e in eng.log if e[0] == "admit"]
    assert admits == sorted(admits)
    out = s.drain()
    assert [rid for rid, _ in out] == [3, 4]


def test_idle_steps_are_not_run_and_drain_terminates():
    s, eng = _sched(4)
    assert s.step(10) == [] and eng.log == []
    assert s.drain() == []
    _submit(s, 0)
    assert [rid for rid, _ in s.drain()] == [0]
    assert sum(e[1] for e in eng.log if e[0] == "run") == N_STEPS


def test_random_traces_against_the_contract():
    rng = np.random.default_rng(0)
    for trial in range(20):
        slots = int(rng.integers(1, 5))
        s, eng = _sched(slots)
        rid, got = 0, []
        for _ in range(int(rng.integers(1, 12))):
            for _ in range(int(rng.integers(0, 4))):
                _submit(s, rid)
                rid += 1
            got += [r for r, _ in s.step(int(rng.integers(1, 8)))]
        got += [r for r, _ in s.drain()]
        assert sorted(got) == list(range(rid))
        # FIFO: requests are admitted in submission order
        admits = [e[2] for e in eng.log if e[0] == "admit"]
        assert admits == list(range(rid))


# ------------------------------------------------------------------------------------------------ refusals
def _model(**over):
    args = default_args(layers=1, diffusion_steps=4, **over)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    return model, diffusion


def test_refusals_before_engine_work():
    model, diffusion = _model()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    # a CPU model has no engine: every refusal below must come first (the engine would raise RuntimeError)
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousSampler(diffusion, cfg, 4, 24, sampler="plms")
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousSampler(diffusion, cfg, 4, 24, sampler="dpm_solver")
    with pytest.raises(ValueError):
        b200mdm.ContinuousSampler(diffusion, cfg, 4, 24, sampler="ddpm", eta=0.5)
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousSampler(diffusion, b200mdm.HandshakeSampleModel(cfg, 2), 4, 24)
    with pytest.raises(TypeError):
        b200mdm.ContinuousSampler(diffusion, torch.nn.Linear(2, 2), 4, 24)
    dip, ddiff = _model(arch="trans_dec", text_encoder_type="bert", pred_len=20, context_len=20)
    with pytest.raises(NotImplementedError):
        b200mdm.ContinuousSampler(ddiff, dip, 4, 40)
    with pytest.raises(RuntimeError):                 # a supported model gets as far as the engine
        b200mdm.ContinuousSampler(diffusion, cfg, 4, 24)


def test_mixed_t_refusals_before_engine_work():
    model, diffusion = _model()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    x = torch.zeros(2, 263, 1, 8)
    t = torch.tensor([0, 2])
    y = dict(scale=torch.ones(2), text_embed=torch.zeros(1, 2, 512))
    with pytest.raises(NotImplementedError):
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": y}, const_noise=True)
    with pytest.raises(NotImplementedError):
        diffusion.ddim_sample(b200mdm.HandshakeSampleModel(cfg, 2), x, t, model_kwargs={"y": y})
    with pytest.raises(NotImplementedError):
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": dict(y, inpainting_mask=x.bool(), inpainted_motion=x)})
    with pytest.raises(NotImplementedError):
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": dict(y, target_cond=torch.zeros(2, 1, 3))})
    dip, ddiff = _model(arch="trans_dec", text_encoder_type="bert", pred_len=8, context_len=8)
    with pytest.raises(NotImplementedError):
        ddiff.p_sample(dip, x, t, model_kwargs={"y": y})
    with pytest.raises(RuntimeError):                 # mixed t itself gets as far as the engine
        diffusion.p_sample(cfg, x, t, model_kwargs={"y": y})
    with pytest.raises(AssertionError):               # p_mean_variance keeps one schedule index per batch
        diffusion.p_mean_variance(cfg, x, t, model_kwargs={"y": y})


# ------------------------------------------------------------------------------------------------ golden fixture
def test_mixed_t_golden_against_the_oracle_per_sample_step():
    """tests/golden/mixed_t_small.npz (the reference's p_sample / ddim_sample at t = (7, 0, 3, 5)) is, row by row, the
    fp32 oracle's step at that row's own index: the reference's step is per sample."""
    from oracle import gen_golden_mixed_t as gm
    from oracle import mdm_oracle as mo
    from oracle import schedule_oracle as so
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "mixed_t_small.npz"))
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=gm.L, seed=1), gm.L)
    tabs = so.diffusion_tables(so.named_betas("cosine", gm.STEPS))
    inp, x, eps = gm.inputs()
    for b, i in enumerate(gm.TS):
        s = slice(b, b + 1)
        with torch.no_grad():
            x0 = mo.cfg_denoise_enc(W, x[s], i, inp["text_embed"][:, s], inp["scale"][s], inp["lengths"][s])
            want = {"ddpm": mo.p_sample_step(tabs, x0, x[s], i, eps[s])[0],
                    "ddim_eta0": mo.ddim_step(tabs, x0, x[s], i, eps[s], 0.0),
                    "ddim_eta0.5": mo.ddim_step(tabs, x0, x[s], i, eps[s], 0.5)}
        for name, w in want.items():
            for key, ref in ((name + "_sample", w), (name + "_pred_xstart", x0)):
                got = torch.from_numpy(g[key][s]).double()
                err = float((got - ref.double()).norm() / ref.double().norm())
                assert err < 1e-5, (b, key, err)
