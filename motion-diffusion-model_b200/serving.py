"""Continuous batching: a fixed batch of slots, each running its own request at its own step (DESIGN.md, "Continuous
batching").

    sampler = b200mdm.ContinuousSampler(diffusion, model, slots=64, nframes=196)
    rid = sampler.submit(text_embed=clip_row, length=120, scale=2.5, seed=7)
    for rid, motion in sampler.step(10): ...      # motions finished in these 10 steps, [njoints, nfeats, length]
    done = sampler.drain()

A request's motion does not depend on the slot it lands in, on what the other slots run, or on when it was admitted:
admitted into slot b with (seed s, sample index g) it is bitwise row b of p_sample_loop / ddim_sample_loop with
noise_seed = s and sample_index_base = g - b at the same batch and frame count, with its conditioning at row b.

ContinuousChainSampler does the same for the BERT-memory decoders: DiP, where every slot runs its own autoregressive
chain of pred_len-frame chunks with its own prompt(s) and prefix, and the plain BERT decoder.

The scheduling lives in SlotScheduler, which only calls slot_admit / slots_run / slot_handoff / slot_read on the engine
it is given.
"""
import collections

import numpy as np
import torch

from . import _lib
from .model.mdm import engine_for
from .utils.sampler_util import resolve

# n_chunks: chunk boundaries of the request (a chain); out: its motion buffer, written at each boundary (None: one
# chunk, read into a new tensor at its end)
_Request = collections.namedtuple("_Request", "rid embed action scale length seed sample_index n_chunks out",
                                  defaults=(1, None))


class SlotScheduler:
    """FIFO admission of queued requests into free slots at step boundaries, and the read-out of finished ones.

    A request runs n_chunks chunks of n_steps steps.  A slot admitted at step boundary k finishes chunk c at boundary
    k + (c + 1) n_steps; the scheduler knows that without asking the device, so it runs the step graph in runs up to
    the next boundary and never polls.  At a boundary that ends one of its chunks but the last, the slot is handed off
    (slot_handoff: the chunk is written out and the next one armed); at the one that ends its last chunk it is read
    (slot_read), and so freed, before any admission there.  Idle steps (no occupied slot) are not run."""

    def __init__(self, engine, slots, n_steps, sample_shape, device, use_graph=True):
        self.engine, self.slots, self.n_steps = engine, int(slots), int(n_steps)
        self.sample_shape, self.device, self.use_graph = tuple(sample_shape), device, use_graph
        self.queue = collections.deque()
        self.occupant = [None] * self.slots         # the _Request in each slot
        self.left = [0] * self.slots                # steps of its current chunk still to run
        self.chunk = [0] * self.slots               # its current chunk

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
                self.occupant[b], self.left[b], self.chunk[b] = r, self.n_steps, 0

    def _boundaries(self, out):
        done = sorted((self.occupant[b].rid, b) for b in range(self.slots)
                      if self.occupant[b] is not None and self.left[b] == 0)
        for rid, b in done:
            r, c = self.occupant[b], self.chunk[b]
            if c + 1 < r.n_chunks:
                self.engine.slot_handoff(b, r, c)
                self.left[b], self.chunk[b] = self.n_steps, c + 1
                continue
            x = r.out if r.out is not None else torch.empty(self.sample_shape, device=self.device, dtype=torch.float32)
            self.engine.slot_read(b, x)
            out.append((rid, x[..., :r.length]))
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
            self._boundaries(out)
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
    this package does not drive (TypeError); BERT-memory decoders take ContinuousChainSampler.  Sampling anything else on the same model ends the session: later calls
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
            raise NotImplementedError("ContinuousSampler does not take BERT text memories (DiP, the BERT decoder): "
                                      "serve them with b200mdm.ContinuousChainSampler")
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


# A chain request's conditioning: its prompts (tokens [n_tokens, C] fp32 and mask [n_tokens] uint8, 1 = padding, on the
# device, one pair or one per chunk) and its prefix [njoints * nfeats, context_len] (None for the plain BERT decoder)
_Chain = collections.namedtuple("_Chain", "tokens masks prefix include_prefix")


class _ChainSlots:
    """The slot protocol of SlotScheduler on an engine's token-memory session (Engine.chain_slot_*): an admission
    arms chunk 0, a hand-off writes chunk c into the request's motion and arms chunk c + 1 (with its own prompt when the
    request has one per chunk), and the read is the hand-off of the last chunk, which frees the slot."""

    def __init__(self, eng):
        self.eng = eng

    def slot_admit(self, slot, chain, action, scale, length, seed, sample_index):
        self.eng.chain_slot_admit(slot, chain.tokens[0], chain.masks[0], chain.prefix, scale, length, chain.include_prefix,
                                  seed, sample_index)

    def slots_run(self, n, use_graph=True):
        self.eng.slots_run(n, use_graph)

    def slot_handoff(self, slot, r, c):
        chain = r.embed
        per_chunk = len(chain.tokens) > 1
        self.eng.chain_slot_handoff(slot, r.out, chain.tokens[c + 1] if per_chunk else None,
                                    chain.masks[c + 1] if per_chunk else None)

    def slot_read(self, slot, out):
        self.eng.chain_slot_handoff(slot, out)
        return out


class ContinuousChainSampler:
    """Continuous batching for the BERT-memory decoders, with DDPM or DDIM (eta) on an MDM or a
    ClassifierFreeSampleModel (guided: every request brings its own scale).

    DiP (context_len > 0): every slot runs its own autoregressive chain of pred_len-frame chunks, with its own prefix
    and its own prompt, or one prompt per chunk.  A request of `length` frames runs ceil(length / pred_len) chunks;
    between them its last context_len frames become its prefix on the device.  Admitted into slot b with (seed s,
    sample index g), its motion is bitwise row b of AutoRegressiveSampler(args, p_sample_loop / ddim_sample_loop,
    required_frames=length).sample(...) with noise_seed = s, sample_index_base = g - b, at the same slots, pred_len,
    context_len and n_tokens, with the request's prefix, tokens, mask and scale at row b (and y['mask'] admitting every
    frame: the length only crops the motion).

    The plain BERT decoder (context_len 0; nframes frames per slot): a request is one chunk without a prefix, and its
    length masks its frames as y['lengths'] does in p_sample_loop.

    n_tokens: the memory width of every slot; a prompt has up to n_tokens tokens and is padded to it.  Refused before
    any engine work: other samplers and the handshake, joint-control and multi-prompt wrappers (NotImplementedError),
    models without a BERT memory (ValueError: they take ContinuousSampler), models this package does not drive
    (TypeError).  Target conditioning and inpainting are not taken by submit.  Sampling anything else on the same model
    ends the session: later calls then raise from the engine."""

    def __init__(self, diffusion, model, slots, *, n_tokens, nframes=None, sampler="ddpm", eta=0.0, clip_denoised=False,
                 use_graph=True):
        if sampler not in ("ddpm", "ddim"):
            raise NotImplementedError("continuous batching runs 'ddpm' and 'ddim' (got %r): PLMS and DPM-Solver++ carry "
                                      "a per-loop history that is not per slot" % (sampler,))
        if sampler == "ddpm" and eta != 0.0:
            raise ValueError("eta is a DDIM parameter")
        if int(slots) <= 0:
            raise ValueError("slots must be positive")
        if not 1 <= int(n_tokens) <= _lib.MAX_MEMORY_TOKENS:
            raise ValueError("n_tokens %d outside 1 .. %d" % (int(n_tokens), _lib.MAX_MEMORY_TOKENS))
        diffusion._check_supported()
        diffusion._refuse(model, "Continuous batching")
        r = resolve(model)
        if r.mdm is not None and not r.mdm.is_dip:
            raise ValueError("ContinuousChainSampler serves the BERT-memory decoders (DiP, humanml_trans_dec_512_bert); "
                             "serve this model with b200mdm.ContinuousSampler")
        m = r.mdm
        if m is not None:
            self.context_len = int(m.context_len)
            if self.context_len > 0:
                if nframes is not None and int(nframes) != m.pred_len:
                    raise ValueError("a DiP slot holds one chunk of pred_len = %d frames (got nframes %d)"
                                     % (m.pred_len, int(nframes)))
                nframes = m.pred_len
            elif nframes is None or int(nframes) <= 0:
                raise ValueError("the plain BERT decoder needs nframes, the frames of a slot")
        eng, guided = engine_for(model)              # TypeError for a model this package does not drive
        self.model, self.mdm, self.guided = model, m, guided
        self.slots, self.nframes, self.n_tokens = int(slots), int(nframes), int(n_tokens)
        self.device = next(m.parameters()).device
        mode = _lib.MODE_DDPM if sampler == "ddpm" else _lib.MODE_DDIM
        eng.set_schedule(diffusion.schedule_rows(eta), diffusion._timestep_map(),
                         key=(id(diffusion), float(eta), diffusion.num_timesteps))
        eng.chain_slots_begin(self.slots, self.nframes, guided, mode, self.n_tokens,
                              _lib.FLAG_CLIP_DENOISED if clip_denoised else 0)
        self.scheduler = SlotScheduler(_ChainSlots(eng), self.slots, diffusion.num_timesteps,
                                       (m.njoints, m.nfeats, self.nframes), self.device, use_graph)
        self._next_id = 0

    @property
    def pending(self):
        """Requests queued and not yet admitted."""
        return self.scheduler.pending

    @property
    def active(self):
        """Slots holding a request."""
        return self.scheduler.active

    def _prompt(self, te):
        """One (tokens, mask) pair -> (tokens [n_tokens, C] fp32, mask [n_tokens] uint8) on the device, padded with zero
        tokens under mask 1.  tokens [Mt, C] or [Mt, 1, C]; mask [Mt] or [1, Mt], True / 1 = padding."""
        if not isinstance(te, (tuple, list)) or len(te) != 2:
            raise ValueError("a prompt's text_embed is a (tokens, mask) pair")
        C = self.mdm.clip_dim
        tok = torch.as_tensor(te[0]).detach().to(device=self.device, dtype=torch.float32).reshape(-1, C)
        msk = torch.as_tensor(te[1]).detach().to(device=self.device).reshape(-1)
        if tok.shape[0] != msk.shape[0]:
            raise ValueError("tokens (%d) and mask (%d) of a prompt differ in length" % (tok.shape[0], msk.shape[0]))
        if not 1 <= tok.shape[0] <= self.n_tokens:
            raise ValueError("a prompt of %d tokens: 1 .. n_tokens = %d" % (tok.shape[0], self.n_tokens))
        tokens = torch.zeros(self.n_tokens, C, device=self.device, dtype=torch.float32)
        mask = torch.ones(self.n_tokens, device=self.device, dtype=torch.uint8)
        tokens[:tok.shape[0]] = tok
        mask[:msk.shape[0]] = (msk != 0).to(torch.uint8)
        return tokens, mask

    def submit(self, text=None, text_embed=None, prefix=None, length=None, include_prefix=False, scale=None, *, seed,
               sample_index=None):
        """Queue one request; returns its id.
        text: a str, or a list of one str per chunk (encoded here by the model's text encoder); or text_embed: a
        (tokens [Mt, C], mask [Mt]) pair, or a list of one pair per chunk (DiP).  prefix [njoints, nfeats, context_len]
        (DiP only, required there).  length: frames of the motion (default nframes; the BERT decoder: at most nframes).
        include_prefix: the motion starts with the prefix, as AutoRegressiveSampler's autoregressive_include_prefix.
        scale: the guidance scale, required by a guided sampler.  sample_index: the global sample index of its Philox
        stream (default: its id).  ValueError, before any engine work, for anything it cannot run."""
        m, T, ctx = self.mdm, self.nframes, self.context_len
        if (text is None) == (text_embed is None):
            raise ValueError("give text or text_embed (one of them)")
        length = T if length is None else int(length)
        if length < 1:
            raise ValueError("length %d < 1" % length)
        if ctx == 0 and length > T:
            raise ValueError("length %d: the plain BERT decoder runs one chunk of at most %d frames" % (length, T))
        n_chunks = -(-length // T) if ctx > 0 else 1
        if text is not None:
            texts = [text] if isinstance(text, str) else list(text)
            prompts = [None] * len(texts)
        else:
            prompts = list(text_embed) if isinstance(text_embed, list) else [text_embed]
        if len(prompts) not in (1, n_chunks):
            raise ValueError("%d prompts for %d chunks: one prompt, or one per chunk" % (len(prompts), n_chunks))
        shape = (m.njoints, m.nfeats, ctx)
        if ctx > 0:
            if prefix is None:
                raise ValueError("a DiP request needs its prefix [%d, %d, %d]" % shape)
            pf = torch.as_tensor(prefix).detach()
            if pf.dim() == 4 and pf.shape[0] == 1:
                pf = pf[0]
            if tuple(pf.shape) != shape:
                raise ValueError("prefix of shape %s: [%d, %d, %d] expected" % ((tuple(pf.shape),) + shape))
            pf = pf.to(device=self.device, dtype=torch.float32).contiguous()
        elif prefix is not None or include_prefix:
            raise ValueError("the plain BERT decoder takes no prefix")
        if self.guided and scale is None:
            raise ValueError("a guided sampler needs each request's scale")
        if not self.guided and scale is not None:
            raise ValueError("scale is for a ClassifierFreeSampleModel")
        if text is not None:
            prompts = [m.encode_text([t]) for t in texts]
        prompts = [self._prompt(te) for te in prompts]
        out = torch.empty(m.njoints, m.nfeats, length, device=self.device, dtype=torch.float32)
        if include_prefix:
            out[..., :min(ctx, length)] = pf[..., :min(ctx, length)]
        chain = _Chain([p[0] for p in prompts], [p[1] for p in prompts],
                       pf.reshape(m.njoints * m.nfeats, ctx) if ctx > 0 else None, bool(include_prefix))
        rid = self._next_id
        self._next_id += 1
        self.scheduler.queue.append(_Request(rid, chain, 0, float(scale) if scale is not None else 0.0, length, int(seed),
                                             rid if sample_index is None else int(sample_index), n_chunks, out))
        return rid

    def step(self, n=1):
        """Advance every occupied slot by n steps, handing chains over and filling free slots from the queue (FIFO) at
        each step boundary; returns the motions finished in the window, [(request id, motion [njoints, nfeats,
        length])], in completion order."""
        return self.scheduler.step(n)

    def drain(self):
        """Run until the queue and all slots are empty."""
        return self.scheduler.drain()
