"""Continuous batching: a fixed batch of slots, each running its own request at its own step (DESIGN.md, "Continuous
batching").

    sampler = b200mdm.ContinuousSampler(diffusion, model, slots=64, nframes=196)
    rid = sampler.submit(text_embed=clip_row, length=120, scale=2.5, seed=7)
    for rid, motion in sampler.step(10): ...      # motions finished in these 10 steps, [njoints, nfeats, length]
    done = sampler.drain()

A request's motion does not depend on the slot it lands in, on what the other slots run, or on when it was admitted:
admitted into slot b with (seed s, sample index g) it is bitwise row b of p_sample_loop / ddim_sample_loop with
noise_seed = s and sample_index_base = g - b at the same batch and frame count, with its conditioning at row b.

The scheduling lives in SlotScheduler, which only calls slot_admit / slots_run / slot_read on the engine it is given.
"""
import collections

import torch

from . import _lib
from .model.mdm import engine_for
from .utils.sampler_util import resolve

_Request = collections.namedtuple("_Request", "rid embed action scale length seed sample_index")


class SlotScheduler:
    """FIFO admission of queued requests into free slots at step boundaries, and the read-out of finished ones.

    A slot admitted at step boundary k finishes at boundary k + n_steps; the scheduler knows that without asking the
    device, so it runs the step graph in runs up to the next finish and never polls.  A finished slot is read (and so
    freed) at the boundary where it finishes, before any admission there.  Idle steps (no occupied slot) are not run."""

    def __init__(self, engine, slots, n_steps, sample_shape, device, use_graph=True):
        self.engine, self.slots, self.n_steps = engine, int(slots), int(n_steps)
        self.sample_shape, self.device, self.use_graph = tuple(sample_shape), device, use_graph
        self.queue = collections.deque()
        self.occupant = [None] * self.slots         # the _Request in each slot
        self.left = [0] * self.slots                # its steps still to run

    @property
    def pending(self):
        return len(self.queue)

    @property
    def active(self):
        return sum(r is not None for r in self.occupant)

    def _admit(self):
        for b in range(self.slots):
            if not self.queue:
                return
            if self.occupant[b] is None:
                r = self.queue.popleft()
                self.engine.slot_admit(b, r.embed, r.action, r.scale, r.length, r.seed, r.sample_index)
                self.occupant[b], self.left[b] = r, self.n_steps

    def _read_finished(self, out):
        done = sorted((self.occupant[b].rid, b) for b in range(self.slots)
                      if self.occupant[b] is not None and self.left[b] == 0)
        for rid, b in done:
            x = torch.empty(self.sample_shape, device=self.device, dtype=torch.float32)
            self.engine.slot_read(b, x)
            out.append((rid, x[..., :self.occupant[b].length]))
            self.occupant[b] = None

    def step(self, n=1):
        """Advance every occupied slot by up to n steps; returns [(request id, motion)] finished in the window, in
        completion order (by request id within one step)."""
        out = []
        k = 0
        while k < n:
            self._admit()
            busy = [self.left[b] for b in range(self.slots) if self.occupant[b] is not None]
            if not busy:
                break
            r = min(n - k, min(busy))
            self.engine.slots_run(r, self.use_graph)
            for b in range(self.slots):
                if self.occupant[b] is not None:
                    self.left[b] -= r
            k += r
            self._read_finished(out)
        return out

    def drain(self):
        """Run until the queue and every slot are empty; returns every motion finished on the way."""
        out = []
        while self.queue or self.active:
            out += self.step(self.n_steps)
        return out


class ContinuousSampler:
    """Continuous batching over `slots` rows of `nframes` frames with DDPM or DDIM (eta) on an MDM or a
    ClassifierFreeSampleModel (guided: every request brings its own scale).  Every request's eps comes from its own
    Philox stream (seed, sample index), so a request is reproducible whatever runs beside it.

    Refused before any engine work: PLMS, DPM-Solver++ and other samplers (NotImplementedError), the handshake,
    joint-control and multi-prompt wrappers (NotImplementedError), BERT-memory decoders (NotImplementedError), and models
    this package does not drive (TypeError).  Sampling anything else on the same model ends the session: later calls
    then raise from the engine."""

    def __init__(self, diffusion, model, slots, nframes, *, sampler="ddpm", eta=0.0, clip_denoised=False, use_graph=True):
        if sampler not in ("ddpm", "ddim"):
            raise NotImplementedError("continuous batching runs 'ddpm' and 'ddim' (got %r): PLMS and DPM-Solver++ carry "
                                      "a per-loop history that is not per slot" % (sampler,))
        if sampler == "ddpm" and eta != 0.0:
            raise ValueError("eta is a DDIM parameter")
        if int(slots) <= 0 or int(nframes) <= 0:
            raise ValueError("slots and nframes must be positive")
        diffusion._check_supported()
        diffusion._refuse(model, "Continuous batching")
        r = resolve(model)
        if r.mdm is not None and r.mdm.is_dip:
            raise NotImplementedError("continuous batching with BERT text memories (DiP, the BERT decoder) is not "
                                      "implemented: their token memories and prefixes are not per slot")
        eng, guided = engine_for(model)              # TypeError for a model this package does not drive
        self.model, self.mdm, self.guided = model, r.mdm, guided
        self.slots, self.nframes = int(slots), int(nframes)
        self.device = next(r.mdm.parameters()).device
        mode = _lib.MODE_DDPM if sampler == "ddpm" else _lib.MODE_DDIM
        eng.set_schedule(diffusion.schedule_rows(eta), diffusion._timestep_map(),
                         key=(id(diffusion), float(eta), diffusion.num_timesteps))
        eng.slots_begin(self.slots, self.nframes, guided, mode, _lib.FLAG_CLIP_DENOISED if clip_denoised else 0)
        self.scheduler = SlotScheduler(eng, self.slots, diffusion.num_timesteps, (r.mdm.njoints, r.mdm.nfeats, self.nframes),
                                       self.device, use_graph)
        self._next_id = 0

    @property
    def pending(self):
        """Requests queued and not yet admitted."""
        return self.scheduler.pending

    @property
    def active(self):
        """Slots holding a request."""
        return self.scheduler.active

    def submit(self, text=None, text_embed=None, action=None, length=None, scale=None, *, seed, sample_index=None):
        """Queue one request; returns its id.  text (encoded here) or text_embed [cond_dim] (or any shape with one row)
        for text models, action for action models; length: frames of the motion (default nframes); scale: the
        guidance scale, required by a guided sampler; sample_index: the global sample index of its Philox stream
        (default: its id)."""
        m = self.mdm
        text_model = "text" in m.cond_mode
        embed = None
        if text is not None and text_embed is not None:
            raise ValueError("give text or text_embed, not both")
        if text_model:
            if text is not None:
                text_embed = m.encode_text([text])
            if text_embed is None:
                raise ValueError("a text-conditioned model needs text or text_embed")
            embed = torch.as_tensor(text_embed).to(device=self.device, dtype=torch.float32).reshape(-1, m.clip_dim)
            if embed.shape[0] != 1:
                raise ValueError("one text embedding per request (got %d rows)" % embed.shape[0])
            embed = embed[0].contiguous()
        elif text is not None or text_embed is not None:
            raise ValueError("the model is not text-conditioned")
        act = -1
        if "action" in m.cond_mode:
            if action is None:
                raise ValueError("an action-conditioned model needs an action")
            act = int(torch.as_tensor(action).reshape(-1)[0])
            if not 0 <= act < m.num_actions:
                raise ValueError("action %d outside [0, %d)" % (act, m.num_actions))
        elif action is not None:
            raise ValueError("the model is not action-conditioned")
        length = self.nframes if length is None else int(length)
        if not 1 <= length <= self.nframes:
            raise ValueError("length %d outside [1, %d]" % (length, self.nframes))
        if self.guided and scale is None:
            raise ValueError("a guided sampler needs each request's scale")
        if not self.guided and scale is not None:
            raise ValueError("scale is for a ClassifierFreeSampleModel")
        rid = self._next_id
        self._next_id += 1
        self.scheduler.queue.append(_Request(rid, embed, max(act, 0), float(scale) if scale is not None else 0.0,
                                             length, int(seed), rid if sample_index is None else int(sample_index)))
        return rid

    def step(self, n=1):
        """Advance every occupied slot by n steps, filling free slots from the queue (FIFO) at each step boundary;
        returns the motions finished in the window, [(request id, motion [njoints, nfeats, length])], in completion
        order."""
        return self.scheduler.step(n)

    def drain(self):
        """Run until the queue and all slots are empty."""
        return self.scheduler.drain()
