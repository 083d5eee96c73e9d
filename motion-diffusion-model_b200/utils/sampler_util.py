"""Sampling-time model wrappers (host mirror of the reference's utils/sampler_util.py)."""
import numpy as np
import torch
import torch.nn as nn

from .misc import wrapped_getattr


class ClassifierFreeSampleModel(nn.Module):
    """Classifier-free guidance wrapper (reference utils/sampler_util.py:10-38).

    The reference deep-copies `y`, runs the denoiser twice and blends
    `out_uncond + scale * (out - out_uncond)`.  Here the cond / uncond pair is packed into ONE batch of 2B inside the
    engine and the blend is applied to the hidden rows in front of the (linear) output projection, which is the same
    expression in exact arithmetic; `y` is never copied or mutated.
    """

    def __init__(self, model):
        super().__init__()
        self.model = model
        assert self.model.cond_mask_prob > 0, \
            "Cannot run a guided diffusion on a model that has not been trained with no conditions"
        self.rot2xyz = self.model.rot2xyz
        self.translation = self.model.translation
        self.njoints = self.model.njoints
        self.nfeats = self.model.nfeats
        self.data_rep = self.model.data_rep
        self.cond_mode = self.model.cond_mode
        self.encode_text = self.model.encode_text

    def forward(self, x, timesteps, y=None):
        assert self.model.cond_mode in ["text", "action"]
        from ..model.mdm import _run_model
        return _run_model(self.model, x, timesteps, y, guided=True)

    def __getattr__(self, name, default=None):
        return wrapped_getattr(self, name, default=None)


def handshake_layout(batch, nframes, handshake_size, lengths=None, motion_start=None):
    """(lengths int64 [batch], motion_start bool [batch]) numpy arrays of a batch of chained windows (DESIGN.md,
    "Long motions from chained windows"): window b has lengths[b] <= nframes frames (all nframes without lengths) and
    begins a new motion where motion_start[b] (without motion_start, the batch is one motion).  ValueError for h < 0, a
    shape mismatch, a length outside [0, nframes], motion_start[0] False, a chained window with fewer than h frames, or a
    window with a predecessor and a successor and fewer than 2h frames (its two handshakes would overlap)."""
    h = int(handshake_size)
    if h < 0:
        raise ValueError("handshake_size must be >= 0 (got %d)" % h)
    n = np.full(batch, nframes, dtype=np.int64) if lengths is None else \
        np.asarray(lengths.detach().cpu() if torch.is_tensor(lengths) else lengths, dtype=np.int64).reshape(-1)
    if motion_start is None:
        ms = np.zeros(batch, dtype=bool)
        ms[0] = True
    else:
        ms = np.asarray(motion_start.detach().cpu() if torch.is_tensor(motion_start) else motion_start).astype(bool).reshape(-1)
    if n.shape != (batch,) or ms.shape != (batch,):
        raise ValueError("lengths and motion_start need one entry per window (batch %d; got %s and %s)"
                         % (batch, n.shape, ms.shape))
    if ((n < 0) | (n > nframes)).any():
        raise ValueError("window lengths must lie in [0, %d] (got %s)" % (nframes, n.tolist()))
    if not ms[0]:
        raise ValueError("motion_start[0] must be True: the first window begins a motion")
    if h > 0:
        chained_prev = ~ms
        chained_next = np.append(~ms[1:], False)
        for b in range(batch):
            if (chained_prev[b] or chained_next[b]) and n[b] < h:
                raise ValueError("window %d is chained but has %d frames < handshake_size %d" % (b, n[b], h))
            if chained_prev[b] and chained_next[b] and n[b] < 2 * h:
                raise ValueError("window %d has %d frames < 2 x handshake_size %d: its two handshakes would overlap"
                                 % (b, n[b], h))
    return n, ms


def _inner_mdm(model):
    from ..model.mdm import MDM
    inner = model.model if isinstance(model, ClassifierFreeSampleModel) else model
    if not isinstance(inner, MDM):
        raise TypeError("HandshakeSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)" % type(model))
    return inner


class HandshakeSampleModel(nn.Module):
    """Long motions from chained windows (DoubleTake's first take, Shafir et al., "Human Motion Diffusion as a
    Generative Prior"), with this project's weights (DESIGN.md): the batch is a list of windows, y['lengths'] their
    lengths and y['motion_start'] (bool [B]) marks the windows that begin a motion (absent: the whole batch is one
    motion).  The last h = handshake_size frames of every window and the first h frames of the next window of the same
    motion are replaced, in the model output, by

        H_j = (1 - a_j) * D[p, n_p - h + j] + a_j * D[b, j],   a_j = (j + 1) / (h + 1),   j = 0 .. h-1,

    so every denoising step forces the two to agree.  `model` is a b200mdm MDM or ClassifierFreeSampleModel; the blend
    runs inside the engine's guidance-blend kernel, in every sampler (DDPM, DDIM, PLMS, DPM-Solver++).  Stitch the
    final windows with `stitch_handshake`.  Prefix-completion (DiP) models, DDIM inversion and the variational bound are
    not supported (NotImplementedError)."""

    def __init__(self, model, handshake_size):
        super().__init__()
        inner = _inner_mdm(model)
        if inner.is_prefix_comp or (inner.arch == "trans_dec" and not inner.emb_trans_dec):
            raise NotImplementedError("handshakes are not implemented for prefix-completion (DiP) models")
        if int(handshake_size) < 0:
            raise ValueError("handshake_size must be >= 0 (got %d)" % int(handshake_size))
        self.model = model
        self.handshake_size = int(handshake_size)
        self.rot2xyz = self.model.rot2xyz
        self.translation = self.model.translation
        self.njoints = self.model.njoints
        self.nfeats = self.model.nfeats
        self.data_rep = self.model.data_rep
        self.cond_mode = self.model.cond_mode
        self.encode_text = self.model.encode_text

    def forward(self, x, timesteps, y=None):
        from ..model.mdm import _run_model
        guided = isinstance(self.model, ClassifierFreeSampleModel)
        if guided:
            assert self.model.model.cond_mode in ["text", "action"]
        return _run_model(_inner_mdm(self.model), x, timesteps, y, guided=guided, handshake=self.handshake_size)

    def __getattr__(self, name, default=None):
        return wrapped_getattr(self, name, default=None)


def stitch_handshake(sample, lengths, handshake_size, motion_start=None):
    """The motions of a batch of chained windows (HandshakeSampleModel): for each motion, its first window's frames
    [:n], then each later window's [h:n].  sample [B, njoints, nfeats, T]; lengths [B] (None: all T); returns a list of
    [njoints, nfeats, L_k] tensors, L_k = sum(n) - (windows - 1) * h."""
    B, T = int(sample.shape[0]), int(sample.shape[-1])
    n, ms = handshake_layout(B, T, handshake_size, lengths, motion_start)
    h = int(handshake_size)
    motions = []
    for b in range(B):
        piece = sample[b, ..., : int(n[b])] if ms[b] else sample[b, ..., h: int(n[b])]
        if ms[b]:
            motions.append([piece])
        else:
            motions[-1].append(piece)
    return [torch.cat(p, dim=-1) for p in motions]


class AutoRegressiveSampler:
    """DiP's outer loop (reference utils/sampler_util.py:41-81): generate `required_frames` as a chain of `pred_len`
    chunks, each a full diffusion loop of the trans_dec engine conditioned on the last `context_len` frames of the
    previous chunk (y['prefix']).  Host control flow only; every chunk is one `sample_fn` call, i.e. one replay of the
    engine's captured step graph per diffusion step.  The caller's kwargs are never mutated (the reference deep-copies
    them per chunk; here only the dicts that change are rebuilt)."""

    def __init__(self, args, sample_fn, required_frames=196):
        self.sample_fn = sample_fn
        self.args = args
        self.required_frames = required_frames

    def sample(self, model, shape, **kargs):
        pred_len, context_len = self.args.pred_len, self.args.context_len
        n_iterations = self.required_frames // pred_len + int(self.required_frames % pred_len > 0)
        y0 = kargs["model_kwargs"]["y"]
        cur_prefix = y0["prefix"].clone()
        dynamic_text_mode = isinstance(y0["text"][0], list) if "text" in y0 else False   # a prompt per chunk
        samples_buf = [cur_prefix] if getattr(self.args, "autoregressive_include_prefix", False) else []
        ar_shape = list(shape)
        ar_shape[-1] = pred_len
        tape = kargs.get("noise_tape")            # b200mdm extension: one tape per chunk, [n_iterations, n_run+1, ...]
        for i in range(n_iterations):
            y = dict(y0)
            y["prefix"] = cur_prefix
            if dynamic_text_mode:
                y["text"] = [s[i] for s in y0["text"]]
                if getattr(model, "text_encoder_type", "bert") != "bert":
                    raise NotImplementedError("DiP model only supports BERT text encoder at the moment.")
                y["text_embed"] = (y0["text_embed"][0][:, :, i], y0["text_embed"][1][:, i])
            cur = dict(kargs)
            cur["model_kwargs"] = dict(kargs["model_kwargs"], y=y)
            if tape is not None:
                cur["noise_tape"] = tape[i]
            if kargs.get("noise") is not None and kargs["noise"].dim() == len(ar_shape) + 1:   # x_T per chunk
                cur["noise"] = kargs["noise"][i]
            sample = self.sample_fn(model, ar_shape, **cur)
            samples_buf.append(sample[..., -pred_len:].clone())
            cur_prefix = sample[..., -context_len:].clone()
        return torch.cat(samples_buf, dim=-1)[..., :self.required_frames]
