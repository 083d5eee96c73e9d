"""GPU: the state the engine keeps between calls, checked against a fresh engine bit for bit.

An engine keeps a captured step graph per workspace (recaptured when its GraphKey changes), a pool of parked workspaces
per (batch, nframes, CFG) with their PLMS eps ring, DPM-Solver++ x0 history and continuation counters, the DiP text
memory sized by n_tokens, schedule tables that move when a longer schedule outgrows them, the target and inpainting
inputs, and its weights.  Every loop below runs on one long-lived engine per model kind (the reused engine), and then
on a fresh engine given only the state that loop needs: schedule, conditioning, target, inpainting, prefix and noise
stream -- or, for a loop continued over several range calls, the same chain of ranges and nothing in between.  The two
results must have the same bits, with and without the step graph.  The first full loop of each (model kind, sampler,
target) is also held to the fp32 oracles within the project's 1e-3 bound, which ties the fresh engine to something
independent.

A small mirror of the documented contract predicts which continuations must fail with B200MDM_ESTATE (another loop on
that workspace, b200mdm_plms_step for PLMS, pool eviction, a weight reload, a different order, a stale table).

  * seq 1-6: scripted sequences, one per test, so a failure names the transition;
  * random walk: ~60 seeded operations per model kind, every loop compared, the operation log printed on failure;
  * caller memory: every entry point that writes caller memory writes a view inside guard bands, and the inputs the ABI
    does not let it alias come back with the same bits;
  * inpainting is the sampler's: b200mdm_denoise ignores it, and b200mdm_set_cond* clears it."""
import ctypes
import importlib
import zlib

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.engine import Engine
from b200mdm.utils.model_util import create_gaussian_diffusion
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import dpm_oracle as do
from oracle import mdm_oracle as mo
from oracle import philox_oracle as px
from oracle import plms_oracle as po
from oracle import reverse_oracle as ro
from oracle import schedule_oracle as so
from oracle import target_oracle as to

pytestmark = pytest.mark.gpu
RTOL = 1e-3
L = 2
TEMB_ROWS = 1200                 # room for the 1100-step schedule, whose tables outgrow the engine's first allocation
SCHEDULES = (6, 10, 1100)
CTX = 8                          # DiP prefix frames
JOINTS = importlib.import_module("motion-diffusion-model_b200.synthetic").HML_TARGET_JOINTS


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def same(a, b):
    """The same bits (NaN payloads and signed zeros included)."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().reshape(-1).view(torch.uint8),
                                                                     b.contiguous().reshape(-1).view(torch.uint8))


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(_seed(*key))


# ------------------------------------------------------------------------------------------------ model kinds
class Kind:
    """One model kind: its engine configuration, weights, oracle and the inputs of each shape (B, T, guided, Mt)."""

    def __init__(self, name, cfg, sd, shapes, target=False):
        self.name, self.cfg, self.sd, self.shapes, self.target = name, cfg, sd, shapes, target
        self.W = mo.OracleWeights(sd, L)
        self.JF = cfg["njoints"] * cfg["nfeats"]
        self._inp, self._tape = {}, {}
        self.full_sd = dict(sd)
        self.full_sd["sequence_pos_encoder.pe"] = so.positional_table(cfg["pos_embed_max_len"], 512)

    def make(self):
        eng = Engine(**self.cfg)
        eng.load_state_dict(self.full_sd)
        return eng

    def xshape(self, s):
        return (s[0], self.cfg["njoints"], self.cfg["nfeats"], s[1])

    def inputs(self, s):
        if s in self._inp:
            return self._inp[s]
        B, T, guided, Mt = s
        rng = np.random.default_rng(_seed(self.name, s))
        lengths = torch.from_numpy(np.concatenate([[T], rng.integers(1, T + 1, B - 1)]).astype(np.int64))
        scale = torch.from_numpy(rng.choice([0.0, 1.0, 2.5, 2.0], B).astype(np.float32))
        y = dict(lengths=lengths.cuda())
        o = dict(lengths=lengths, scale=scale if guided else None)
        if guided:
            y["scale"] = scale.cuda()
        if self.name == "a2m":
            action = torch.from_numpy(rng.integers(0, 12, (B, 1)).astype(np.int64))
            y["action"], o["action"] = action.cuda(), action
        elif self.name == "dip":
            enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, CTX, seed=int(rng.integers(1 << 30)))
            y["text_embed"], y["prefix"] = (enc.cuda(), tmask.cuda()), prefix.cuda()
            o.update(enc=enc, tmask=tmask, prefix=prefix)
        else:
            te = torch.from_numpy(rng.standard_normal((1, B, 512)).astype(np.float32))
            y["text_embed"], o["cond"] = te.cuda(), te
        tg = b200mdm.synthetic_target_inputs(B, seed=int(rng.integers(1 << 30))) if self.target else None
        g = torch.Generator(device="cuda").manual_seed(int(rng.integers(1 << 30)))
        shape = self.xshape(s)
        inp = dict(
            y=y, o=o, tg=tg,
            x=[torch.randn(shape, device="cuda", generator=g) for _ in range(2)],
            ts=torch.from_numpy(rng.integers(0, 1000, B).astype(np.int32)),
            # two inpainting pairs (mask uint8, motion); the tensors live as long as the module: an engine may hold them
            inpaint=[((torch.rand(shape, device="cuda", generator=g) < 0.3).to(torch.uint8),
                      torch.rand(shape, device="cuda", generator=g) * 1.8 - 0.9) for _ in range(2)])
        self._inp[s] = inp
        return inp

    def tape(self, s, first, n):
        k = (s, first, n)
        if k not in self._tape:
            self._tape[k] = torch.randn((n,) + self.xshape(s), device="cuda", generator=_gen(self.name, k))
        return self._tape[k]

    # oracle denoiser f(x, i) for the conditioning of shape s
    def denoiser(self, s, target, tmap):
        o, W = self.inputs(s)["o"], self.W
        g = None
        if target:
            tg = self.inputs(s)["tg"]
            valid = to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"])
            g = to.target_embedding(W, "single", tg["target_cond"], valid, 1)
        if self.name == "enc":
            if g is None:
                return po.enc_denoiser(W, tmap, o["cond"], o["scale"], o["lengths"])
            if o["scale"] is None:
                return lambda x, i: to.denoise_enc(W, x, int(tmap[i]), o["cond"], g, o["lengths"])
            return lambda x, i: to.cfg(to.denoise_enc, o["scale"], W, x, int(tmap[i]), o["cond"], g, o["lengths"])
        if self.name == "a2m":
            return lambda x, i: mo.denoise_enc(W, x, int(tmap[i]), None, o["lengths"], True, False, o["action"])
        if self.name == "dip":
            if o["scale"] is None:
                return lambda x, i: mo.denoise_dec(W, x, int(tmap[i]), o["enc"], o["tmask"], o["prefix"], o["lengths"])
            return po.dec_denoiser(W, tmap, o["enc"], o["tmask"], o["prefix"], o["scale"], o["lengths"])
        return deo.denoiser(W, tmap, o["cond"], o["scale"], o["lengths"], g=g)


def _cfg(**over):
    c = dict(arch="trans_enc", latent_dim=512, ff_size=1024, num_layers=L, num_heads=4, njoints=263, nfeats=1,
             cond_mode="text", cond_dim=512, num_actions=1, mask_frames=True, pos_embed_max_len=5000,
             temb_rows=TEMB_ROWS)
    c.update(over)
    return c


_KINDS = {}


def kind(name):
    if name in _KINDS:
        return _KINDS[name]
    sdf = b200mdm.synthetic_state_dict
    tgt = dict(target_encoder="single", target_enc_layers=1, target_joint_names=JOINTS)
    if name == "enc":
        k = Kind(name, _cfg(**tgt), sdf(num_layers=L, seed=61, target_encoder="single"),
                 [(3, 24, True, None), (2, 16, True, None), (4, 24, True, None), (3, 24, False, None), (1, 40, True, None)],
                 target=True)
    elif name == "a2m":
        k = Kind(name, _cfg(njoints=25, nfeats=6, cond_mode="action", num_actions=12),
                 sdf(num_layers=L, seed=62, input_feats=150, cond_mode="action", num_actions=12),
                 [(3, 20, False, None), (2, 30, False, None), (4, 20, False, None), (1, 20, False, None), (3, 30, False, None)])
    elif name == "dip":
        k = Kind(name, _cfg(arch="trans_dec", cond_dim=768, context_len=CTX, dec_memory=_lib.DEC_MEMORY_TOKENS),
                 sdf(arch="trans_dec", num_layers=L, cond_dim=768, seed=63),
                 [(2, 16, True, 16), (2, 16, True, 33), (3, 20, True, 7), (2, 24, False, 65), (1, 16, True, 150)])
    else:
        k = Kind(name, _cfg(arch="trans_dec", emb_trans_dec=True, dec_memory=_lib.DEC_MEMORY_CLIP, **tgt),
                 sdf(arch="trans_dec", num_layers=L, cond_dim=512, seed=64, target_encoder="single"),
                 [(3, 24, True, None), (2, 16, True, None), (4, 24, True, None), (3, 24, False, None), (1, 40, True, None)],
                 target=True)
    _KINDS[name] = k
    return k


KINDS = ["enc", "a2m", "dip", "clipdec"]


class Sched:
    def __init__(self, n):
        self.n = n
        d = create_gaussian_diffusion(default_args(layers=L, diffusion_steps=n))
        self.rows, self.next, self.dpm, self.tmap = d.schedule_rows(0.0), d.schedule_next_rows(), d.schedule_dpm_rows(), \
            list(range(n))
        self._tables = None

    def tables(self):
        if self._tables is None:
            self._tables = so.diffusion_tables(so.named_betas("cosine", self.n))
        return self._tables


_SCHED = {}


def sched(n):
    if n not in _SCHED:
        _SCHED[n] = Sched(n)
    return _SCHED[n]


# ------------------------------------------------------------------------------------------------ calls shared by both engines
def do_set_cond(eng, k, s):
    inp = k.inputs(s)
    eng.set_cond(s[0], s[1], inp["y"], s[2], torch.device("cuda"))


def do_set_target(eng, k, s):
    tg = k.inputs(s)["tg"]
    eng._set_target(s[0], dict(target_cond=tg["target_cond"], target_joint_names=tg["target_joint_names"],
                               is_heading=tg["is_heading"]), torch.device("cuda"))


def do_set_inpaint(eng, pair):
    _lib.check(eng.lib.b200mdm_set_inpaint(eng.h, _p(pair[0]) if pair else None, _p(pair[1]) if pair else None))


def do_set_schedule(eng, n, tables=True):
    sc = sched(n)
    eng.set_schedule(sc.rows, sc.tmap)
    if tables:
        eng.set_schedule_next(sc.next)
        eng.set_schedule_dpm(sc.dpm)


MODES = {"ddpm": _lib.MODE_DDPM, "ddpm_philox": _lib.MODE_DDPM, "ddim": _lib.MODE_DDIM}


def do_range(eng, k, s, spec, x_in, x_out, use_graph):
    """spec = (sampler, order, first_index, n_run, flags)."""
    sampler, order, first, n, flags = spec
    if sampler in ("ddpm", "ddim"):
        eng.sample_loop_range(MODES[sampler], first, n, x_in, x_out, k.tape(s, first, n), flags, use_graph)
    elif sampler == "ddpm_philox":
        eng.sample_loop_range(MODES[sampler], first, n, x_in, x_out, None, flags, use_graph)
    elif sampler == "plms":
        eng.plms_loop_range(order, first, n, x_in, x_out, flags, use_graph)
    elif sampler == "dpm":
        eng.dpm_loop_range(order, first, n, x_in, x_out, flags, use_graph)
    else:
        eng.ddim_reverse_loop_range(first, n, x_in, x_out, flags, use_graph)


# ------------------------------------------------------------------------------------------------ the clean room
class Ctx(tuple):
    """(shape, target on, inpainting (shape, pair index, contents version) or None, schedule length, noise seed)."""


_CLEAN = {}
_ORACLE_DONE = set()


def _apply_ctx(eng, k, ctx, prev):
    s, target, inp, n, seed = ctx
    if prev is None or prev[3] != n:
        do_set_schedule(eng, n)
    if prev is None or prev[:3] != ctx[:3]:
        do_set_cond(eng, k, s)
        if target:
            do_set_target(eng, k, s)
        if inp is not None:
            do_set_inpaint(eng, k.inputs(inp[0])["inpaint"][inp[1]])
    if seed is not None:
        eng.set_noise_stream(seed, 0)


def clean_loop(k, chain, use_graph):
    """The result of `chain` [(ctx, spec, x index), ...] (a loop and the ranges continuing it) on a fresh engine."""
    key = (k.name, tuple(chain), use_graph)
    if key in _CLEAN:
        return _CLEAN[key]
    eng = k.make()
    try:
        prev = None
        s = chain[0][0][0]
        out = torch.empty(k.xshape(s), device="cuda")
        for j, (ctx, spec, xi) in enumerate(chain):
            _apply_ctx(eng, k, ctx, prev)
            prev = ctx
            do_range(eng, k, s, spec, k.inputs(s)["x"][xi] if j == 0 else None, out if j == len(chain) - 1 else None,
                     use_graph)
        torch.cuda.synchronize()
    finally:
        eng.close()
    _CLEAN[key] = out
    if len(chain) == 1:
        _oracle_check(k, chain[0], out)
    return out


def _oracle_check(k, link, out):
    """The first full loop of each (kind, sampler, target) on a small schedule, without the clamp: the fp32 oracle."""
    (s, target, inp, n, seed), (sampler, order, first, nrun, flags), xi = link
    full = (first == 0 and nrun == n) if sampler == "rev" else (first == n - 1 and nrun == n)
    tag = (k.name, sampler, order, target)
    if not full or flags or n > 10 or tag in _ORACLE_DONE:
        return
    _ORACLE_DONE.add(tag)
    sc = sched(n)
    f = k.denoiser(s, target, sc.tmap)
    x = k.inputs(s)["x"][xi].cpu()
    ip = None
    if inp is not None:
        m, mo_ = k.inputs(inp[0])["inpaint"][inp[1]]
        ip = (m.bool().cpu(), mo_.cpu())
    tabs = sc.tables()
    if sampler in ("ddpm", "ddim"):
        tape = [x] + list(k.tape(s, first, nrun).cpu())
        ref = deo.sample_loop(f, tabs, tape, sampler, inpaint=ip)
    elif sampler == "ddpm_philox":
        B = s[0]
        eps = [torch.from_numpy(px.normal(B, k.JF * s[1], seed, 0, i)).reshape(x.shape) for i in range(n - 1, -1, -1)]
        ref = deo.sample_loop(f, tabs, [x] + eps, "ddpm", inpaint=ip)
    elif sampler == "plms":
        ref = po.plms_loop(f, tabs, x, order, inpaint=ip)
    elif sampler == "dpm":
        ref = do.dpm_loop(f, tabs, x, order, inpaint=ip)
    else:
        ref = ro.reverse_loop(f, tabs, x, 0, n, inpaint=ip)
    e = rel_err(out, ref)
    print("fresh engine vs the fp32 oracle, %s %s order %d target %s: %.2e" % (k.name, sampler, order, target, e))
    assert e < RTOL, (tag, e)


def clean_denoise(k, ctx):
    key = (k.name, "denoise", ctx)
    if key not in _CLEAN:
        eng = k.make()
        try:
            s = ctx[0]
            _apply_ctx(eng, k, ctx, None)
            inp = k.inputs(s)
            _CLEAN[key] = eng.denoise(inp["x"][0], inp["ts"])
            torch.cuda.synchronize()
        finally:
            eng.close()
    return _CLEAN[key]


# ------------------------------------------------------------------------------------------------ the reused engine
class Reused:
    """The long-lived engine of a kind, with a mirror of what the contract says it holds: the current conditioning,
    target, inpainting, schedule and noise seed, the pool of workspaces (LRU, current + 3 parked) and each workspace's
    open PLMS / DPM-Solver++ chain."""
    MAX_PARKED = 3

    def __init__(self, k):
        self.k = k
        self.eng = k.make()
        self.log = []
        self.reset_mirror()
        self.n = None
        self.fresh_next = self.fresh_dpm = False
        self.seed = None

    def reset_mirror(self):
        self.cur, self.pool, self.clock = None, {}, 0      # pool: workspace key -> last use
        self.ws = {}                                        # workspace key -> {"plms": chain, "dpm": chain}
        self.s = None
        self.target = False
        self.inp = None

    def note(self, *op):
        self.log.append(" ".join(str(o) for o in op))

    def fail_msg(self):
        return "operation log (%s):\n  %s" % (self.k.name, "\n  ".join(self.log))

    # --- state
    def set_cond(self, s):
        self.note("set_cond", s)
        do_set_cond(self.eng, self.k, s)
        w = s[:3]
        self.clock += 1
        if w != self.cur:
            if self.cur is not None:
                self.pool[self.cur] = self.clock
            if w in self.pool:
                del self.pool[w]
            else:
                while len(self.pool) > self.MAX_PARKED:
                    lru = min(self.pool, key=self.pool.get)
                    del self.pool[lru]
                    self.ws.pop(lru, None)
                self.ws[w] = {"plms": None, "dpm": None}
            self.cur = w
        self.s, self.target, self.inp = s, False, None

    def set_target(self, on=True):
        self.note("set_target" if on else "set_cond (clears the target)")
        if on:
            do_set_target(self.eng, self.k, self.s)
            self.target = True
        else:
            self.set_cond(self.s)

    def set_inpaint(self, which, version=0):
        """which: pair index of the current shape, or None to clear."""
        self.note("set_inpaint", which, version)
        pair = self.k.inputs(self.s)["inpaint"][which] if which is not None else None
        do_set_inpaint(self.eng, pair)
        self.inp = (self.s, which, version) if which is not None else None

    def set_schedule(self, n, tables=True):
        self.note("set_schedule", n, "with tables" if tables else "without the reverse / DPM tables")
        do_set_schedule(self.eng, n, tables)
        self.n, self.fresh_next, self.fresh_dpm = n, tables, tables

    def set_tables(self):
        self.note("set_schedule_next + set_schedule_dpm")
        self.eng.set_schedule_next(sched(self.n).next)
        self.eng.set_schedule_dpm(sched(self.n).dpm)
        self.fresh_next = self.fresh_dpm = True

    def set_noise(self, seed):
        self.note("set_noise_stream", seed)
        self.eng.set_noise_stream(seed, 0)
        self.seed = seed

    def reload(self):
        self.note("reload weights")
        self.eng.load_state_dict(self.k.full_sd)
        self.reset_mirror()

    def ctx(self, sampler):
        return Ctx((self.s, self.target, self.inp, self.n, self.seed if sampler == "ddpm_philox" else None))

    # --- predictions of the contract
    def can_continue(self, sampler, order):
        ch = self.ws[self.cur][sampler]
        if ch is None or ch[-1][1][1] != order or ch[0][0][3] != self.n:
            return False
        if sampler == "dpm" and not self.fresh_dpm:
            return False
        last = ch[-1][1]
        return last[2] - last[3] >= 0

    def expected_error(self, sampler, order, fresh):
        if sampler == "rev" and not self.fresh_next:
            return _lib.ESTATE
        if sampler == "dpm" and not self.fresh_dpm:
            return _lib.ESTATE
        if not fresh:
            ch = self.ws[self.cur][sampler]
            if ch is None or ch[-1][1][1] != order:
                return _lib.ESTATE
        return None

    def try_continue(self, sampler, order, n, **kw):
        """Continue the workspace's open chain where the mirror says it may be continued; where the contract refuses
        (no chain, another order, a stale table), check that the engine refuses with ESTATE.  A chain that has reached
        index 0, or was opened under another schedule, is left alone."""
        if self.can_continue(sampler, order):
            last = self.ws[self.cur][sampler][-1][1]
            return self.loop(sampler, order, n=min(n, last[2] - last[3] + 1), cont=True, flags=last[4], **kw)
        if self.expected_error(sampler, order, False) == _lib.ESTATE:
            return self.loop(sampler, order, first=self.n - 1, n=1, cont=True, **kw)
        return None

    # --- loops
    def loop(self, sampler, order=0, first=None, n=None, xi=0, flags=0, use_graph=True, cont=False, expect=None,
             leave=False):
        """One loop or range on the reused engine, compared with the clean room.  cont: continue the open chain of the
        workspace (first defaults to the next index); leave: x_out NULL, the result stays in the engine (the next range
        of the chain is compared).  Returns the result, or the error code when one is expected."""
        s = self.s
        if cont:
            last = self.ws[self.cur].get(sampler)
            if first is None:
                first = last[-1][1][2] - last[-1][1][3] if last else self.n - 1
        elif first is None:
            first = 0 if sampler == "rev" else self.n - 1
        if n is None:
            n = (self.n - first) if sampler == "rev" else first + 1
        spec = (sampler, order, first, n, flags)
        self.note("loop", spec, "continue" if cont else "x%d" % xi, "graph" if use_graph else "eager")
        want = self.expected_error(sampler, order, not cont) if expect is None else expect
        out = torch.full(self.k.xshape(s), float("nan"), device="cuda")
        x_in = None if cont else self.k.inputs(s)["x"][xi]
        if want is not None:
            with pytest.raises(_lib.B200MDMError) as exc:
                do_range(self.eng, self.k, s, spec, x_in, out, use_graph)
                torch.cuda.synchronize()
            assert exc.value.code == want, self.fail_msg()
            self.note("  -> error %d as the contract says" % want)
            return want
        do_range(self.eng, self.k, s, spec, x_in, None if leave else out, use_graph)
        torch.cuda.synchronize()
        link = (self.ctx(sampler), spec, xi)
        w = self.ws[self.cur]
        if sampler in ("plms", "dpm"):
            chain = (w[sampler] + [link]) if cont else [link]
        else:
            chain = [link]
        w["plms"] = w["dpm"] = None            # any loop ends the open chain of the workspace ...
        if sampler in ("plms", "dpm"):
            w[sampler] = chain                 # ... and a PLMS / DPM loop opens its own
        if leave:
            return None
        ref = clean_loop(self.k, tuple(chain), use_graph)
        assert same(out, ref), "%s differs from a fresh engine (max |diff| %.3e)\n%s" % (
            spec, (out - ref).abs().max().item(), self.fail_msg())
        return out

    def denoise(self):
        self.note("denoise")
        inp = self.k.inputs(self.s)
        out = self.eng.denoise(inp["x"][0], inp["ts"])
        torch.cuda.synchronize()
        ref = clean_denoise(self.k, Ctx((self.s, self.target, None, self.n, None)))
        assert same(out, ref), "denoise differs from a fresh engine\n" + self.fail_msg()
        return out

    def sample_step(self, mode=_lib.MODE_DDIM, index=0):
        self.note("sample_step", mode, index)
        inp = self.k.inputs(self.s)
        x, pred = self.eng.sample_step(mode, index, inp["x"][1], inp["x"][0])
        torch.cuda.synchronize()
        return x, pred

    def plms_step(self, index, order):
        self.note("plms_step", index, order)
        inp = self.k.inputs(self.s)
        r = self.eng.plms_step(index, order, inp["x"][1], [inp["x"][0]])
        torch.cuda.synchronize()
        self.ws[self.cur]["plms"] = None
        return r


_REUSED = {}


def reused(name):
    """One reused engine per kind for the whole module: every test leaves state behind for the next one."""
    if name not in _REUSED:
        _REUSED[name] = Reused(kind(name))
    return _REUSED[name]


# ------------------------------------------------------------------------------------------------ scripted sequences
@pytest.mark.parametrize("name", KINDS)
def test_seq1_interleaved_samplers(name):
    """DDIM -> PLMS 4 -> PLMS 2 -> DDPM (tape) -> DPM 2M -> DDIM inversion -> DDPM (Philox) -> DDIM on one workspace, each
    graph recaptured on a GraphKey change; then the same sequence eagerly."""
    r = reused(name)
    r.set_schedule(6)
    r.set_cond(r.k.shapes[0])
    r.set_noise(1234)
    for use_graph in (True, False):
        for sampler, order in (("ddim", 0), ("plms", 4), ("plms", 2), ("ddpm", 0), ("dpm", 2), ("rev", 0),
                               ("ddpm_philox", 0), ("ddim", 0), ("dpm", 1), ("plms", 3)):
            r.loop(sampler, order, use_graph=use_graph)
    if r.k.target:
        r.set_target()
        for sampler, order in (("ddim", 0), ("ddpm", 0), ("plms", 2), ("dpm", 2), ("rev", 0)):
            r.loop(sampler, order)


@pytest.mark.parametrize("name", KINDS)
def test_seq2_continuation_through_interruptions(name):
    """A PLMS order-3 loop and a DPM 2M loop split into ranges, with a denoise, a sample_step and a loop on another
    workspace (then set_cond back) between them: the stitched result is the uninterrupted loop, bit for bit."""
    r = reused(name)
    k = r.k
    r.set_schedule(10)
    a, b = k.shapes[0], k.shapes[2]                       # two (B, T, CFG) workspaces
    for sampler, order in (("plms", 3), ("dpm", 2)):
        for use_graph in (True, False):
            r.set_cond(a)
            whole = r.loop(sampler, order, use_graph=use_graph)
            r.loop(sampler, order, first=9, n=3, use_graph=use_graph, leave=True)
            r.denoise()
            r.loop(sampler, order, n=2, cont=True, use_graph=use_graph)
            r.sample_step(_lib.MODE_DDIM, 4)
            r.sample_step(_lib.MODE_DDPM, 7)
            r.loop(sampler, order, n=2, cont=True, use_graph=use_graph)
            r.set_cond(b)
            r.loop("ddim", use_graph=use_graph)
            r.loop(sampler, order, use_graph=use_graph)            # the other workspace's own loop of this kind
            r.set_cond(a)                                          # back: the parked workspace keeps its loop
            last = r.loop(sampler, order, n=3, cont=True, use_graph=use_graph)
            assert same(last, whole), "the stitched %s loop differs from the whole loop\n%s" % (sampler, r.fail_msg())
    # dpm_pred_xstart: the x0 of the last step -- at i = 0 the sample itself, above it the DDIM x0 of the same forward
    x0 = torch.empty_like(last)
    r.eng.dpm_pred_xstart(x0)
    torch.cuda.synchronize()
    assert same(x0, last)
    x3 = clean_loop(k, ((r.ctx("dpm"), ("dpm", 2, 9, 3, 0), 0),), True)
    r.loop("dpm", 2, first=9, n=4)
    r.eng.dpm_pred_xstart(x0)
    _, pred = r.eng.sample_step(_lib.MODE_DDIM, 6, x3, k.tape(a, 9, 4)[0])
    torch.cuda.synchronize()
    assert same(x0, pred), "dpm_pred_xstart is not the x0 of the loop's last step"
    # where continuation must fail with ESTATE
    r.set_cond(a)
    for sampler, order, other in (("plms", 3, 2), ("dpm", 2, 1)):
        r.loop(sampler, order, first=9, n=3)
        r.loop(sampler, other, n=2, cont=True, expect=_lib.ESTATE)            # a different order
        r.loop(sampler, order, n=2, cont=True)                                # ... which does not end the loop
        r.loop("ddim")                                                        # a DDIM loop on the same workspace
        r.loop(sampler, order, n=2, cont=True, expect=_lib.ESTATE)
        r.loop(sampler, order, first=9, n=3)
        r.reload()                                                            # a weight reload
        r.set_cond(a)
        r.loop(sampler, order, n=2, cont=True, expect=_lib.ESTATE)
    r.loop("plms", 3, first=9, n=3)
    r.plms_step(5, 3)                                                         # b200mdm_plms_step
    r.loop("plms", 3, n=2, cont=True, expect=_lib.ESTATE)


@pytest.mark.parametrize("name", KINDS)
def test_seq3_pool_eviction(name):
    """Six (B, T, CFG) triples in turn, each left holding a PLMS ring, a DPM history or a reverse-mode graph, so LRU
    frees some of them; then every triple again: continuations where the workspace survived, ESTATE where it did not,
    and a fresh loop either way."""
    r = reused(name)
    k = r.k
    r.set_schedule(6)
    extra = [(5, 12, k.shapes[0][2], k.shapes[0][3]), (2, 12, k.shapes[1][2], k.shapes[1][3])]
    triples = k.shapes[:4] + extra
    kinds = [("plms", 2), ("dpm", 2), ("rev", 0)]
    for j, s in enumerate(triples):
        r.set_cond(s)
        sampler, order = kinds[j % 3]
        if sampler == "rev":
            r.loop(sampler, order)
        else:
            r.loop(sampler, order, first=5, n=2)
    for j, s in enumerate(triples + triples[:2]):
        r.set_cond(s)
        sampler, order = kinds[j % 3]
        if sampler != "rev":
            r.try_continue(sampler, order, 2)
        r.loop(kinds[(j + 1) % 3][0], kinds[(j + 1) % 3][1], use_graph=j % 2 == 0)


@pytest.mark.parametrize("name", KINDS)
def test_seq4_schedule_moves(name):
    """Park workspaces holding PLMS, DPM and reverse graphs, grow the schedule past the tables' capacity (they move and
    every graph is dropped), come back to the small schedule: each parked workspace's next loop matches.  Reverse and
    DPM loops between set_schedule and their own table are refused."""
    r = reused(name)
    k = r.k
    r.set_schedule(10)
    parked = [(k.shapes[0], "plms", 2), (k.shapes[1], "dpm", 2), (k.shapes[2], "rev", 0)]
    for s, sampler, order in parked:
        r.set_cond(s)
        r.loop(sampler, order, first=9 if sampler != "rev" else 0, n=3)
    r.set_schedule(1100, tables=False)
    r.loop("dpm", 2, first=1099, n=2, expect=_lib.ESTATE)
    r.loop("rev", 0, first=0, n=2, expect=_lib.ESTATE)
    r.loop("ddim", first=1099, n=2)
    r.set_tables()
    r.loop("dpm", 2, first=1099, n=2)
    r.loop("rev", 0, first=1096, n=3)
    r.loop("ddpm", first=2, n=3, use_graph=False)
    r.set_schedule(10, tables=False)
    for s, sampler, order in parked:
        r.set_cond(s)
        if sampler != "plms":
            r.loop(sampler, order, first=9 if sampler == "dpm" else 0, n=2, expect=_lib.ESTATE)
    r.set_tables()
    for s, sampler, order in parked:
        r.set_cond(s)
        if sampler == "rev":
            r.loop("rev", 0, first=0, n=10)
        else:
            # a chain opened under this schedule is not ended by the excursion (unless LRU evicted its workspace)
            r.try_continue(sampler, order, 2)
            r.loop(sampler, order)


def test_seq5_dip_memory_length():
    """n_tokens 16 -> 150 -> 16 -> 33 -> 64 -> 65 -> 7 in one (B, T, CFG) workspace with a captured graph: every
    cross-attention dispatch (<= 16, <= 32, <= 64, long) and back."""
    r = reused("dip")
    r.set_schedule(6)
    for j, mt in enumerate((16, 150, 16, 33, 64, 65, 7)):
        r.set_cond((2, 16, True, mt))
        r.loop("ddim", use_graph=True)
        r.loop("dpm", 2, use_graph=j % 2 == 0)
    r.set_cond((2, 16, True, 64))
    r.loop("plms", 2, first=5, n=3)
    r.set_cond((2, 16, True, 65))          # same workspace, another memory: the PLMS loop continues under the new one
    r.loop("plms", 2, n=3, cont=True)


@pytest.mark.parametrize("name", ["enc", "clipdec"])
def test_seq6_target_then_set_cond(name):
    """set_target, loop, set_cond at the same shape, loop: the second loop has no target."""
    r = reused(name)
    r.set_schedule(6)
    s = r.k.shapes[0]
    for use_graph in (True, False):
        r.set_cond(s)
        r.set_target()
        with_t = r.loop("ddim", use_graph=use_graph)
        r.set_cond(s)
        without = r.loop("ddim", use_graph=use_graph)
        assert not same(with_t, without)
        r.set_target()
        assert same(r.loop("ddim", use_graph=use_graph), with_t)


@pytest.mark.parametrize("name", KINDS)
def test_seq6_inpainting_transitions(name):
    """Inpainting set, cleared, set again at a new address, and the same address with new contents; then set_cond at
    the same shape with no new set_inpaint (the loop has none)."""
    r = reused(name)
    r.set_schedule(6)
    s = r.k.shapes[0]
    r.set_cond(s)
    pairs = r.k.inputs(s)["inpaint"]
    saved = pairs[1][1].clone()
    try:
        for sampler, order in (("ddim", 0), ("dpm", 2), ("plms", 2)):
            outs = [r.loop(sampler, order)]
            r.set_inpaint(0)
            outs.append(r.loop(sampler, order))
            r.set_inpaint(None)
            assert same(r.loop(sampler, order), outs[0])
            r.set_inpaint(1)
            outs.append(r.loop(sampler, order))
            pairs[1][1].mul_(-1.0)                                # same address, new contents
            r.set_inpaint(1, version=1)
            outs.append(r.loop(sampler, order))
            pairs[1][1].copy_(saved)
            r.set_inpaint(1, version=0)
            r.set_cond(s)                                         # no set_inpaint: the loop has none
            assert same(r.loop(sampler, order), outs[0])
            for i in range(len(outs)):
                for j in range(i):
                    assert not same(outs[i], outs[j]), (sampler, i, j)
    finally:
        pairs[1][1].copy_(saved)


# ------------------------------------------------------------------------------------------------ inpainting regressions
@pytest.mark.parametrize("name", KINDS)
def test_denoise_ignores_inpainting(name):
    """b200mdm_denoise is model(x, t, y): the sampler's inpainting (p_mean_variance) is not part of it."""
    r = reused(name)
    r.set_schedule(6)
    s = r.k.shapes[0]
    r.set_cond(s)
    bare = r.denoise()
    r.set_inpaint(0)
    assert same(r.denoise(), bare), r.fail_msg()
    inp = r.k.inputs(s)
    x, pred = r.eng.sample_step(_lib.MODE_DDIM, 3, inp["x"][0], inp["x"][1])   # the sampler's x0 keeps it
    torch.cuda.synchronize()
    m, motion = inp["inpaint"][0]
    assert torch.equal(pred[m.bool()], motion[m.bool()])
    r.set_inpaint(None)


@pytest.mark.parametrize("name", KINDS)
def test_set_cond_clears_inpainting(name):
    """A loop after set_cond at the same shape, with no new set_inpaint, equals a fresh engine without inpainting."""
    r = reused(name)
    r.set_schedule(6)
    s = r.k.shapes[0]
    r.set_cond(s)
    r.set_inpaint(1)
    r.loop("ddpm")
    r.set_cond(s)
    assert r.inp is None
    plain = r.loop("ddpm")                       # compared with the clean room, which has no inpainting
    r.set_inpaint(1)
    assert not same(r.loop("ddpm"), plain)


# ------------------------------------------------------------------------------------------------ seeded random walk
@pytest.mark.parametrize("name", KINDS)
def test_random_walk(name):
    r = reused(name)
    k = r.k
    rng = np.random.default_rng({"enc": 1, "a2m": 2, "dip": 3, "clipdec": 4}[name])
    r.set_schedule(6)
    r.set_cond(k.shapes[0])
    r.set_noise(7)
    samplers = [("ddpm", 0), ("ddpm_philox", 0), ("ddim", 0), ("plms", 2), ("plms", 3), ("plms", 4), ("dpm", 1),
                ("dpm", 2), ("rev", 0)]
    try:
        for _ in range(60):
            op = rng.choice(["cond", "target", "inpaint", "sched", "noise", "loop", "loop", "loop", "cont", "denoise",
                             "reload"], p=[.14, .06, .08, .06, .04, .16, .16, .12, .12, .04, .02])
            if op == "cond":
                r.set_cond(k.shapes[rng.integers(5)])
            elif op == "target":
                if k.target:
                    r.set_target(bool(rng.integers(2)))
            elif op == "inpaint":
                r.set_inpaint([None, 0, 1][rng.integers(3)])
            elif op == "sched":
                r.set_schedule(int(rng.choice(SCHEDULES)))
            elif op == "noise":
                r.set_noise(int(rng.integers(1 << 40)))
            elif op == "denoise":
                r.denoise()
            elif op == "reload":
                r.reload()
                r.set_cond(k.shapes[rng.integers(5)])
            elif op in ("loop", "cont"):
                sampler, order = samplers[rng.integers(len(samplers))]
                ug = bool(rng.integers(2))
                flags = _lib.FLAG_CLIP_DENOISED if rng.random() < 0.2 else 0
                if sampler in ("ddpm", "ddpm_philox", "ddim") and rng.random() < 0.2:
                    flags |= _lib.FLAG_CONST_NOISE
                if op == "cont" and sampler in ("plms", "dpm"):
                    r.try_continue(sampler, order, int(rng.integers(1, 5)), use_graph=ug)
                    continue
                n = r.n
                if n > 10:                                             # the long schedule: short ranges only
                    first = int(rng.integers(0, n - 4)) if sampler == "rev" else int(rng.integers(3, n))
                    r.loop(sampler, order, first=first, n=3, xi=int(rng.integers(2)), flags=flags, use_graph=ug)
                elif rng.random() < 0.3 and sampler != "rev":
                    r.loop(sampler, order, first=n - 1, n=int(rng.integers(1, n)), xi=int(rng.integers(2)), flags=flags,
                           use_graph=ug)
                else:
                    r.loop(sampler, order, xi=int(rng.integers(2)), flags=flags, use_graph=ug)
    except AssertionError:
        print(r.fail_msg())
        raise


# ------------------------------------------------------------------------------------------------ caller memory
GUARD = 4096                     # fp32 words on each side
PATTERN = 0x7FA5C3E1             # a NaN bit pattern nothing computes


def guarded(n):
    buf = torch.full((GUARD + n + GUARD,), PATTERN, dtype=torch.int32, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(torch.float32)


def guards_intact(buf, n):
    torch.cuda.synchronize()
    return bool((buf[:GUARD] == PATTERN).all()) and bool((buf[GUARD + n:] == PATTERN).all())


@pytest.mark.parametrize("name", KINDS)
def test_caller_memory_footprint(name):
    r = reused(name)
    k, eng, lib = r.k, r.eng, r.eng.lib
    r.set_schedule(6)
    s = (3, 23, k.shapes[0][2], k.shapes[0][3])          # 23 frames: odd sizes everywhere
    r.set_cond(s)
    if k.target:
        r.set_target()
    inp = k.inputs(s)
    r.set_inpaint(0)
    shape = k.xshape(s)
    n = int(np.prod(shape))
    x, x1 = inp["x"]
    tape = k.tape(s, 5, 6)
    keep = {"x_T": x, "x1": x1, "tape": tape, "mask": inp["inpaint"][0][0], "motion": inp["inpaint"][0][1]}
    y = inp["y"]
    if name == "dip":
        keep.update(enc=y["text_embed"][0], prefix=y["prefix"])
    elif "text_embed" in y:
        keep["text_embed"] = y["text_embed"]
    if k.target:
        keep["target"] = inp["tg"]["target_cond"]
    before = {kk: v.clone() for kk, v in keep.items()}
    ts = np.ascontiguousarray(inp["ts"].numpy())
    tsp = ts.ctypes.data_as(ctypes.c_void_p)
    st = _stream()

    def views(count=1):
        return [guarded(n) for _ in range(count)]

    checks = []
    (b0, o0), = views()
    _lib.check(lib.b200mdm_denoise(eng.h, _p(x), tsp, _p(o0), st))
    checks.append(("denoise out", b0))
    (b0, o0), (b1, o1) = views(2)
    _lib.check(lib.b200mdm_sample_step(eng.h, _lib.MODE_DDPM, 4, _p(x), _p(tape[0]), 0, _p(o0), _p(o1), st))
    checks += [("sample_step x_out", b0), ("sample_step pred_xstart", b1)]
    (b0, o0), = views()
    _lib.check(lib.b200mdm_sample_loop_range(eng.h, _lib.MODE_DDPM, 5, 6, _p(x), _p(o0), _p(tape), n, 0, 1, st))
    checks.append(("sample_loop_range out", b0))
    (b0, o0), (b1, o1), (b2, o2) = views(3)
    old = (ctypes.c_void_p * 1)(x1.data_ptr())
    _lib.check(lib.b200mdm_plms_step(eng.h, 3, 2, _p(x), old, 1, 0, _p(o0), _p(o1), _p(o2), st))
    checks += [("plms_step out", b0), ("plms_step pred", b1), ("plms_step eps_out", b2)]
    _lib.check(lib.b200mdm_dpm_loop_range(eng.h, 2, 5, 3, _p(x), None, 0, 1, st))
    (b0, o0), = views()
    _lib.check(lib.b200mdm_dpm_pred_xstart(eng.h, _p(o0), st))
    checks.append(("dpm_pred_xstart", b0))
    (b0, o0), = views()
    _lib.check(lib.b200mdm_ddim_reverse_loop_range(eng.h, 0, 4, _p(x), _p(o0), 0, 1, st))
    checks.append(("reverse loop out", b0))
    per = k.JF * s[1]
    assert per % 4 != 0
    bp, op = guarded(s[0] * per)
    _lib.check(lib.b200mdm_philox_normal(_p(op), s[0], per, ctypes.c_uint64(99), 5, 2, st))
    torch.cuda.synchronize()
    assert guards_intact(bp, s[0] * per), "philox_normal wrote outside [batch, n_per_sample]"
    want = px.normal(s[0], per, 99, 5, 2)          # logf / sincospif differ from numpy in the last ulp
    assert np.abs(op.cpu().numpy().reshape(s[0], per) - want).max() < 2e-6
    bq, oq = guarded(n)
    _lib.check(lib.b200mdm_q_sample(eng.h, ctypes.c_float(0.6), ctypes.c_float(0.8), _p(x), _p(tape[1]), _p(oq), n, st))
    checks.append(("q_sample out", bq))
    for what, b in checks:
        assert guards_intact(b, n), "%s: a guard word changed" % what
        assert bool((b[GUARD:GUARD + n] != PATTERN).all()), "%s: not every element was written" % what
    for kk, v in keep.items():
        assert same(v, before[kk]), "%s changed" % kk
    r.set_inpaint(None)


def test_table_setters_before_set_schedule():
    """set_schedule_next / _dpm / _vb with a key on a fresh engine, before any set_schedule: each is refused with the
    engine's ESTATE; after set_schedule the same calls upload."""
    eng = Engine(**_cfg())
    s = sched(6)
    vb = create_gaussian_diffusion(default_args(layers=L, diffusion_steps=6)).schedule_vb_rows()
    calls = ((eng.set_schedule_next, s.next), (eng.set_schedule_dpm, s.dpm), (eng.set_schedule_vb, vb))
    for setter, rows in calls:
        with pytest.raises(_lib.B200MDMError) as exc:
            setter(rows, key="k")
        assert exc.value.code == _lib.ESTATE, exc.value
        assert "b200mdm_set_schedule has not been called" in str(exc.value)
    eng.set_schedule(s.rows, s.tmap)
    for setter, rows in calls:
        setter(rows, key="k")
    eng.close()


def test_recover_from_ric_strided_output():
    """recover_from_ric into a strided view (padded rows and samples) inside guard bands: it writes exactly the
    (b, t, joint, axis) elements, each where the strides say."""
    lib = _lib.load()
    B, T, J = 3, 23, 22
    g = torch.Generator(device="cuda").manual_seed(5)
    data = torch.randn(B, 263, T, device="cuda", generator=g) * 0.3
    ref = torch.empty(B, T, J * 3, device="cuda")
    st = _stream()
    _lib.check(lib.b200mdm_recover_from_ric(_p(data), 263 * T, T, 1, None, None, _p(ref), T * J * 3, J * 3, 1, B, T, J, st))
    osc, ost = 2, 2 * J * 3 + 5
    osb = T * ost + 7
    span = (B - 1) * osb + (T - 1) * ost + (3 * J - 1) * osc + 1
    buf, view = guarded(span)
    _lib.check(lib.b200mdm_recover_from_ric(_p(data), 263 * T, T, 1, None, None, _p(view), osb, ost, osc, B, T, J, st))
    torch.cuda.synchronize()
    assert guards_intact(buf, span)
    idx = (torch.arange(B)[:, None, None] * osb + torch.arange(T)[None, :, None] * ost +
           torch.arange(3 * J)[None, None, :] * osc).reshape(-1).cuda()
    written = torch.zeros(span, dtype=torch.bool, device="cuda")
    written[idx] = True
    assert bool((buf[GUARD:GUARD + span][~written] == PATTERN).all()), "an element between the strided rows changed"
    assert same(view[idx].reshape(B, T, 3 * J), ref)
