"""Sampling-time model wrappers (host mirror of the reference's utils/sampler_util.py)."""
from typing import NamedTuple, Optional

import numpy as np
import torch
import torch.nn as nn

from ..model.mdm import MDM, _run_model
from .misc import wrapped_getattr
from .scene import SceneGrid


class _SampleWrapper(nn.Module):
    """A sampling-time wrapper of `model`, registered as the submodule `model`: the attributes the reference's callers
    read are copied from it and every other attribute is looked up on it.  `kind` names a feature wrapper (resolve)."""
    kind = None

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.rot2xyz = self.model.rot2xyz
        self.translation = self.model.translation
        self.njoints = self.model.njoints
        self.nfeats = self.model.nfeats
        self.data_rep = self.model.data_rep
        self.cond_mode = self.model.cond_mode
        self.encode_text = self.model.encode_text

    def __getattr__(self, name, default=None):
        return wrapped_getattr(self, name, default=None)


class ClassifierFreeSampleModel(_SampleWrapper):
    """Classifier-free guidance wrapper (reference utils/sampler_util.py:10-38).

    The reference deep-copies `y`, runs the denoiser twice and blends
    `out_uncond + scale * (out - out_uncond)`.  Here the cond / uncond pair is packed into ONE batch of 2B inside the
    engine and the blend is applied to the hidden rows in front of the (linear) output projection, which is the same
    expression in exact arithmetic; `y` is never copied or mutated.
    """

    def __init__(self, model):
        assert model.cond_mask_prob > 0, \
            "Cannot run a guided diffusion on a model that has not been trained with no conditions"
        super().__init__(model)

    def forward(self, x, timesteps, y=None):
        assert self.model.cond_mode in ["text", "action"]
        return _run_model(self.model, x, timesteps, y, guided=True)


def _core(model):
    """(mdm, guided) of a b200mdm MDM or of a ClassifierFreeSampleModel of one, else None."""
    if isinstance(model, ClassifierFreeSampleModel):
        return (model.model, True) if isinstance(model.model, MDM) else None
    return (model, False) if isinstance(model, MDM) else None


class Resolved(NamedTuple):
    """The wrapper stack a sampler was given (resolve)."""
    mdm: Optional[MDM]          # None: the stack does not end in a model of this package
    guided: bool                # classifier-free guidance
    wrapper: Optional[nn.Module]
    kind: Optional[str]         # wrapper.kind: "handshake", "joint" or "multi"
    core: object                # what the feature wrapper wraps; the model itself without one


def resolve(model):
    """The stack of a model given to a sampler: respace._WrappedModel layers, at most one feature wrapper
    (HandshakeSampleModel, JointControlSampleModel or MultiPromptSampleModel), an optional ClassifierFreeSampleModel
    and an MDM.  Only this package's classes are looked through (model.mdm.engine_for says why): any other object
    gives mdm None."""
    from ..diffusion.respace import _WrappedModel            # respace -> gaussian_diffusion -> this module
    while isinstance(model, _WrappedModel):
        model = model.model
    wrapper = model if isinstance(model, _SampleWrapper) and model.kind is not None else None
    core = model if wrapper is None else wrapper.model
    mdm, guided = _core(core) or (None, False)
    return Resolved(mdm, guided, wrapper, None if wrapper is None else wrapper.kind, core)


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


class HandshakeSampleModel(_SampleWrapper):
    """Long motions from chained windows (DoubleTake's first take, Shafir et al., "Human Motion Diffusion as a
    Generative Prior"), with this project's weights (DESIGN.md): the batch is a list of windows, y['lengths'] their
    lengths and y['motion_start'] (bool [B]) marks the windows that begin a motion (absent: the whole batch is one
    motion).  The last h = handshake_size frames of every window and the first h frames of the next window of the same
    motion are replaced, in the model output, by

        H_j = (1 - a_j) * D[p, n_p - h + j] + a_j * D[b, j],   a_j = (j + 1) / (h + 1),   j = 0 .. h-1,

    so every denoising step forces the two to agree.  `model` is a b200mdm MDM or ClassifierFreeSampleModel; the blend
    runs inside the engine's guidance-blend kernel, in every sampler (DDPM, DDIM, PLMS, DPM-Solver++).  Stitch the
    final windows with `stitch_handshake`.  Every model the engine runs is supported, the BERT decoder (context_len 0)
    included; prefix-completion (DiP, context_len > 0) models, DDIM inversion and the variational bound are not
    (NotImplementedError)."""
    kind = "handshake"

    def __init__(self, model, handshake_size):
        core = _core(model)
        if core is None:
            raise TypeError("HandshakeSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)" % type(model))
        if core[0].is_prefix_comp:
            raise NotImplementedError("handshakes are not implemented for prefix-completion (DiP) models")
        if int(handshake_size) < 0:
            raise ValueError("handshake_size must be >= 0 (got %d)" % int(handshake_size))
        super().__init__(model)
        self.handshake_size = int(handshake_size)

    def forward(self, x, timesteps, y=None):
        mdm, guided = _core(self.model)
        if guided:
            assert mdm.cond_mode in ["text", "action"]
        return _run_model(mdm, x, timesteps, y, guided=guided, wrapper=self)


class JointControlSampleModel(_SampleWrapper):
    """Joint-position control (this project's definition, DESIGN.md "Joint-position control"): at every DDPM / DDIM step
    the model's x0 (after classifier-free guidance) takes `n_iters` gradient steps of size `step_size` on

        G(x0) = 1/2 sum_{t,j} y['joint_weight'][b,j,t] * |recover_from_ric(x0 * std + mean)[t,j] - y['joint_target'][b,j,:,t]|^2,

    before inpainting, the clamp of clip_denoised and the update.  y['joint_target'] [B, J, 3, T] is in sample_to_xyz's
    layout and units; y['joint_weight'] [B, J, T] (float >= 0, or bool) is 0 where a joint is free.  `model` is a b200mdm
    MDM or ClassifierFreeSampleModel of HumanML3D (263 features, J = 22) or KIT (251, J = 21); mean / std [D] are the
    dataset's normalisation.  p_sample_loop, ddim_sample_loop (any eta), their _progressive forms, p_sample and
    ddim_sample honour it, for every model the engine runs (the BERT decoder with context_len 0 included); the other
    samplers, prefix-completion (DiP, context_len > 0) models and AutoRegressiveSampler raise
    NotImplementedError, HandshakeSampleModel and refine_transitions TypeError.  Calling the wrapper is the plain model:
    the guidance belongs to the sampler, as inpainting does.

    Foot contact and floor (DESIGN.md "Joint-position control", "Foot contact and floor"): `contact_weight` adds
    1/2 contact_weight sum_{k,t} kappa[b,k,t] |p[t+1, f_k] - p[t, f_k]|^2 over the four foot joints f_k of the contact
    features (HumanML3D 7, 10, 8, 11; KIT 19, 20, 14, 15), kappa = y['foot_contact'] [B, 4, T] (float >= 0 or bool) or,
    without it, 1 where the step's own de-normalised x0 has contact feature k > 0.5 at frame t and t + 1 < lengths[b];
    `floor_weight` adds 1/2 floor_weight sum_{t < lengths[b], j} min(p[t,j].y - floor_height, 0)^2.  With either weight
    > 0, y['joint_target'] / y['joint_weight'] are optional (absent: no joint term).

    Scene (DESIGN.md "Joint-position control", "Scene: obstacles and uneven ground"): `obstacle_weight` adds
    1/2 obstacle_weight sum_{t < lengths[b], j} max(obstacle_margin - S(p[t,j].x, p[t,j].z), 0)^2 with S = y['obstacle_sdf'],
    a SceneGrid of the obstacles' 2D signed distance (positive outside; SceneGrid.from_shapes builds it for discs and
    boxes), and y['terrain'], a SceneGrid of heights, raises the floor to floor_height + H(p.x, p.z).  Either grid is
    shared by the batch or has one grid per sample.  With obstacle_weight > 0, y['joint_target'] / y['joint_weight'] are
    optional.

    Several characters in one scene (DESIGN.md "Joint-position control", "Several characters in one scene"): with
    `characters` = C >= 2 the batch is B / C scenes, motions [sC, sC + C) forming scene s.  y['scene_placement'] [B, 3]
    (x, z, phi) places each motion's own frame in its scene, Q = rot(phi) p + (x, 0, z) with rot(phi) (x, z) =
    (x cos phi - z sin phi, x sin phi + z cos phi); the other terms keep reading the own frame.  `interaction_weight`
    adds 1/2 interaction_weight sum_{a<b} sum_{t<L_ab} sum_{j,k} max(interaction_margin - |Q_a[t,j] - Q_b[t,k]|, 0)^2 over
    each scene's pairs, L_ab = min(lengths[a], lengths[b]); the reach rows y['interaction_pairs'] int [N, 4] (scene-local
    a, j, b, k with a != b), y['interaction_reach'] [N] and y['interaction_pair_weight'] [N, T] (every scene) or
    [B / C, N, T] add 1/2 sum_n sum_{t<L_ab} w_n[t] max(|Q_a[t,j] - Q_b[t,k]| - reach_n, 0)^2.  With C >= 2,
    y['joint_target'] / y['joint_weight'] are optional."""
    kind = "joint"

    def __init__(self, model, mean, std, step_size, n_iters, *, contact_weight=0.0, floor_weight=0.0, floor_height=0.0,
                 obstacle_weight=0.0, obstacle_margin=0.0, characters=1, interaction_weight=0.0, interaction_margin=0.0):
        core = _core(model)
        if core is None:
            raise TypeError("JointControlSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)" % type(model))
        inner = core[0]
        D = int(inner.njoints) * int(inner.nfeats)
        if inner.data_rep != "hml_vec" or int(inner.nfeats) != 1 or D not in (263, 251):
            raise ValueError("joint-position control needs the ric features of HumanML3D (263) or KIT (251); this model "
                             "has data_rep %r with %d x %d features" % (inner.data_rep, inner.njoints, inner.nfeats))
        if inner.is_prefix_comp:
            raise NotImplementedError("joint-position control is not implemented for prefix-completion (DiP) models")
        step, iters = float(step_size), n_iters
        if not (np.isfinite(step) and step > 0):
            raise ValueError("step_size must be finite and > 0 (got %r)" % step_size)
        if isinstance(iters, bool) or not isinstance(iters, (int, np.integer)) or not 1 <= iters <= 10000:
            raise ValueError("n_iters must be an integer in 1 .. 10000 (got %r)" % (n_iters,))
        mean, std = (torch.as_tensor(np.asarray(v.detach().cpu() if torch.is_tensor(v) else v, dtype=np.float32)).reshape(-1)
                     for v in (mean, std))
        if mean.shape != (D,) or std.shape != (D,):
            raise ValueError("mean and std need %d entries (got %s and %s)" % (D, tuple(mean.shape), tuple(std.shape)))
        cw, fw, fh = float(contact_weight), float(floor_weight), float(floor_height)
        if not (np.isfinite(cw) and cw >= 0 and np.isfinite(fw) and fw >= 0):
            raise ValueError("contact_weight and floor_weight must be finite and >= 0 (got %r, %r)" % (contact_weight, floor_weight))
        if not np.isfinite(fh):
            raise ValueError("floor_height must be finite (got %r)" % (floor_height,))
        ow, om = float(obstacle_weight), float(obstacle_margin)
        if not (np.isfinite(ow) and ow >= 0 and np.isfinite(om) and om >= 0):
            raise ValueError("obstacle_weight and obstacle_margin must be finite and >= 0 (got %r, %r)"
                             % (obstacle_weight, obstacle_margin))
        if isinstance(characters, bool) or not isinstance(characters, (int, np.integer)) or not 1 <= characters <= 8:
            raise ValueError("characters must be an integer in 1 .. 8 (got %r)" % (characters,))
        iw, im = float(interaction_weight), float(interaction_margin)
        if not (np.isfinite(iw) and iw >= 0 and np.isfinite(im) and im >= 0):
            raise ValueError("interaction_weight and interaction_margin must be finite and >= 0 (got %r, %r)"
                             % (interaction_weight, interaction_margin))
        if characters == 1 and iw > 0:
            raise ValueError("interaction_weight > 0 needs characters >= 2")
        super().__init__(model)
        self.mean, self.std = mean, std
        self.step_size, self.n_iters = step, int(iters)
        self.n_joints = 22 if D == 263 else 21
        self.contact_weight, self.floor_weight, self.floor_height = cw, fw, fh
        self.obstacle_weight, self.obstacle_margin = ow, om
        self.characters, self.interaction_weight, self.interaction_margin = int(characters), iw, im

    @property
    def foot(self):
        """True when the foot-contact or floor term is on"""
        return self.contact_weight > 0 or self.floor_weight > 0

    def targets(self, y, shape):
        """(target [B, J, 3, T], weight [B, J, T]) fp32 of y for a sample of `shape`; y is not modified.  ValueError for a
        missing key, a shape other than these, a weight that is negative or not finite, or a target that is not finite
        where its weight is not 0."""
        B, T, J = int(shape[0]), int(shape[-1]), self.n_joints
        if (self.foot or self.obstacle_weight > 0 or self.characters > 1) and "joint_target" not in y and "joint_weight" not in y:
            return torch.zeros(B, J, 3, T), torch.zeros(B, J, T)      # no joint term: a target the kernel never reads
        if "joint_target" not in y or "joint_weight" not in y:
            raise ValueError("JointControlSampleModel needs y['joint_target'] [B, %d, 3, T] and y['joint_weight'] [B, %d, T]"
                             % (J, J))
        c, w = y["joint_target"], y["joint_weight"]
        if not torch.is_tensor(c) or not torch.is_tensor(w):
            raise ValueError("y['joint_target'] and y['joint_weight'] must be tensors")
        if tuple(c.shape) != (B, J, 3, T) or tuple(w.shape) != (B, J, T):
            raise ValueError("y['joint_target'] %s / y['joint_weight'] %s must be %s / %s" % (
                tuple(c.shape), tuple(w.shape), (B, J, 3, T), (B, J, T)))
        if w.dtype != torch.bool and not w.is_floating_point():
            raise ValueError("y['joint_weight'] must be a float or bool tensor")
        w = w.to(torch.float32)
        c = c.to(torch.float32)
        if not bool((torch.isfinite(w) & (w >= 0)).all()):
            raise ValueError("y['joint_weight'] must be finite and >= 0")
        if not bool((torch.isfinite(c) | (w == 0)[:, :, None, :]).all()):
            raise ValueError("y['joint_target'] must be finite where y['joint_weight'] is not 0")
        return c, w

    def foot_contact(self, y, shape):
        """kappa [B, 4, T] fp32 of y['foot_contact'], or None (absent: derived from each step's x0); y is not modified.
        ValueError for a shape other than [B, 4, T], a dtype other than float or bool, or a value that is negative or
        not finite."""
        if not self.foot or y.get("foot_contact") is None:
            return None
        k = y["foot_contact"]
        B, T = int(shape[0]), int(shape[-1])
        if not torch.is_tensor(k) or tuple(k.shape) != (B, 4, T):
            raise ValueError("y['foot_contact'] must be a tensor of shape %s (got %s)"
                             % ((B, 4, T), tuple(k.shape) if torch.is_tensor(k) else type(k)))
        if k.dtype != torch.bool and not k.is_floating_point():
            raise ValueError("y['foot_contact'] must be a float or bool tensor")
        k = k.to(torch.float32)
        if not bool((torch.isfinite(k) & (k >= 0)).all()):
            raise ValueError("y['foot_contact'] must be finite and >= 0")
        return k

    def scene(self, y, shape):
        """(obstacle sdf, terrain) of y, each a SceneGrid or None, or None when no scene term applies; y is not
        modified.  y['obstacle_sdf'] is read when obstacle_weight > 0, y['terrain'] when present.  ValueError for an
        obstacle weight without y['obstacle_sdf'], a terrain with floor_weight 0, a value that is not a SceneGrid, or a
        per-sample grid whose batch is not the sample's."""
        B = int(shape[0])
        sdf = y.get("obstacle_sdf") if self.obstacle_weight > 0 else None
        terrain = y.get("terrain")
        if self.obstacle_weight > 0 and sdf is None:
            raise ValueError("obstacle_weight > 0 needs y['obstacle_sdf'] (a SceneGrid)")
        if terrain is not None and self.floor_weight == 0:
            raise ValueError("y['terrain'] needs floor_weight > 0")
        for name, g in (("obstacle_sdf", sdf), ("terrain", terrain)):
            if g is None:
                continue
            if not isinstance(g, SceneGrid):
                raise ValueError("y[%r] must be a b200mdm.SceneGrid (got %r)" % (name, type(g)))
            if g.per_sample and g.values.shape[0] != B:
                raise ValueError("y[%r] has %d grids for %d samples" % (name, g.values.shape[0], B))
        return None if sdf is None and terrain is None else (sdf, terrain)

    def interaction(self, y, shape):
        """(placement [B, 3], pairs int64 [N, 4] or None, reach [N] or None, pair weight [N, T] / [B / C, N, T] or None)
        fp32 of y, or None with one character per scene; y is not modified.  ValueError for a batch that is not a whole
        number of scenes, a missing or misshaped placement, reach rows without their reach or weights, a row outside
        the scene or its joints or with a == b, or a reach or weight that is negative or not finite."""
        keys = ("scene_placement", "interaction_pairs", "interaction_reach", "interaction_pair_weight")
        if self.characters == 1:
            if any(k in y for k in keys):
                raise ValueError("y[%r] needs characters >= 2" % next(k for k in keys if k in y))
            return None
        B, T, C, J = int(shape[0]), int(shape[-1]), self.characters, self.n_joints
        if B % C:
            raise ValueError("a batch of %d motions is not a whole number of %d-character scenes" % (B, C))
        pl = y.get("scene_placement")
        if not torch.is_tensor(pl) or tuple(pl.shape) != (B, 3) or not pl.is_floating_point():
            raise ValueError("characters >= 2 needs y['scene_placement'], a float tensor [%d, 3] (x, z, phi)" % B)
        pl = pl.to(torch.float32)
        if not bool(torch.isfinite(pl).all()):
            raise ValueError("y['scene_placement'] must be finite")
        if y.get("interaction_pairs") is None:
            return pl, None, None, None
        pairs, reach, pw = y["interaction_pairs"], y.get("interaction_reach"), y.get("interaction_pair_weight")
        pairs = torch.as_tensor(pairs)
        if pairs.dim() != 2 or pairs.shape[1] != 4 or pairs.is_floating_point() or pairs.dtype == torch.bool:
            raise ValueError("y['interaction_pairs'] must be an integer tensor [N, 4] (got %s)" % (tuple(pairs.shape),))
        N = int(pairs.shape[0])
        if not 1 <= N <= 1024:
            raise ValueError("y['interaction_pairs'] holds 1 .. 1024 rows (got %d)" % N)
        pairs = pairs.to(torch.int64).cpu()
        a, j, b, k = pairs.unbind(1)
        if bool(((a < 0) | (a >= C) | (b < 0) | (b >= C) | (a == b) | (j < 0) | (j >= J) | (k < 0) | (k >= J)).any()):
            raise ValueError("y['interaction_pairs'] rows (a, j, b, k) need 0 <= a, b < %d, a != b and 0 <= j, k < %d"
                             % (C, J))
        if not torch.is_tensor(reach) or tuple(reach.shape) != (N,) or not reach.is_floating_point():
            raise ValueError("y['interaction_pairs'] needs y['interaction_reach'], a float tensor [%d]" % N)
        if not torch.is_tensor(pw) or tuple(pw.shape) not in ((N, T), (B // C, N, T)) or not pw.is_floating_point():
            raise ValueError("y['interaction_pairs'] needs y['interaction_pair_weight'], a float tensor %s or %s"
                             % ((N, T), (B // C, N, T)))
        reach, pw = reach.to(torch.float32), pw.to(torch.float32)
        if not bool((torch.isfinite(reach) & (reach >= 0)).all()) or not bool((torch.isfinite(pw) & (pw >= 0)).all()):
            raise ValueError("y['interaction_reach'] and y['interaction_pair_weight'] must be finite and >= 0")
        return pl, pairs, reach, pw

    def forward(self, x, timesteps, y=None):
        return self.model(x, timesteps, y)


# HumanML3D's 263 features per frame: root yaw velocity, root XZ velocity, root height (4), then for the 21 non-root
# joints their root-relative positions (3 each) and rotations (6 each), for all 22 joints their velocities (3 each), and
# 4 foot contacts.  The lower body is the pelvis, hips, knees, ankles and feet; the root features and foot contacts
# belong to it.
_HML_JOINTS = 22
_HML_LOWER_JOINTS = (0, 1, 2, 4, 5, 7, 8, 10, 11)


def body_part_mask(parts):
    """bool [263] feature mask of HumanML3D's body parts: 'lower' or 'upper' (the reference's HML_LOWER_BODY_MASK /
    HML_UPPER_BODY_MASK, which partition the features), or a list of them (their union)."""
    names = [parts] if isinstance(parts, str) else list(parts)
    if not names or any(p not in ("lower", "upper") for p in names):
        raise ValueError("body parts are 'lower' and 'upper' (got %r)" % (parts,))
    low = np.isin(np.arange(_HML_JOINTS), _HML_LOWER_JOINTS)
    lower = np.concatenate([np.ones(4, bool), low[1:].repeat(3), low[1:].repeat(6), low.repeat(3), np.ones(4, bool)])
    out = np.zeros(263, dtype=bool)
    for p in names:
        out |= lower if p == "lower" else ~lower
    return torch.from_numpy(out)


class MultiPromptSampleModel(_SampleWrapper):
    """Multi-prompt guidance (this project's definition, DESIGN.md "Multi-prompt guidance"): K prompts per motion,
    composed around the unconditional prediction as

        x0[b, f, t] = x0_u[b, f, t] + sum_k y['prompt_weight'][b, k, f, t] * (x0_k[b, f, t] - x0_u[b, f, t])

    in fp32, before inpainting, the clamp of clip_denoised and the update.  A body-part prompt is a weight that is
    nonzero on that part's features only (body_part_mask), a time-varying prompt a weight that changes with t, a negative
    prompt a negative weight; K = 1 with the weight y['scale'][b] is ClassifierFreeSampleModel's formula.

    `model` is a b200mdm MDM: trans_enc with CLIP text or action conditioning, the CLIP decoder with a timestep token, or
    the BERT decoder with context_len 0 (prefix-completion (DiP, context_len > 0) models raise NotImplementedError, any
    wrapper TypeError).  y carries the prompts as y['prompt_embed'] fp32 [K, B, C] (for the BERT decoder a list of K
    (tokens [Mt_k, B, 768], padding mask [B, Mt_k]) pairs as encode_text returns them, padded here to the longest) or
    y['prompt_text'] (B lists of K strings, which the sampler encodes into it, one prompt at a time), or
    y['prompt_action'] [B, K] for action models, and y['prompt_weight'] float [B, K, D, T] (either of the last two may
    be 1: it is broadcast, never materialised).  The BERT decoder's unconditional prediction admits every token some
    prompt admits (with K = 1, prompt 0's mask).  lengths, mask, inpainting and target keys keep their meaning;
    y['text'], y['text_embed'] and y['scale'] are not read.  Every sampler but calc_bpd_loop (NotImplementedError)
    honours it; calling the wrapper returns the composed x0."""
    kind = "multi"

    def __init__(self, model):
        if not isinstance(model, MDM):
            raise TypeError("MultiPromptSampleModel wraps a b200mdm MDM (got %r)" % type(model))
        assert model.cond_mask_prob > 0, \
            "Cannot run a guided diffusion on a model that has not been trained with no conditions"
        if model.is_prefix_comp:
            raise NotImplementedError("multi-prompt guidance is not implemented for prefix-completion (DiP) models")
        if model.cond_mode not in ("text", "action"):
            raise ValueError("multi-prompt guidance needs a text- or action-conditioned model (cond_mode %r)"
                             % model.cond_mode)
        super().__init__(model)

    def prompts(self, y, shape):
        """(embed [K, B, C] (a list of K (tokens, mask) pairs for the BERT decoder) or None, action int64 numpy [B, K] or
        None, weight fp32 [B, K, D or 1, T or 1]) of y for a sample of `shape`; y is not modified, and y['prompt_text']
        is not encoded (embed is None for it).  ValueError for a missing or mis-shaped key, K outside 1 .. MAX_PROMPTS,
        a memory outside 1 .. MAX_MEMORY_TOKENS tokens, an action outside the model's classes, or a weight that is not
        finite."""
        from .. import _lib
        B, T = int(shape[0]), int(shape[-1])
        D = int(self.model.njoints) * int(self.model.nfeats)
        w = y.get("prompt_weight")
        if not torch.is_tensor(w) or not w.is_floating_point() or w.dim() != 4:
            raise ValueError("MultiPromptSampleModel needs y['prompt_weight'], a float tensor [B, K, D, T]")
        K = int(w.shape[1])
        if not 1 <= K <= _lib.MAX_PROMPTS:
            raise ValueError("the prompt count K = %d must lie in 1 .. %d" % (K, _lib.MAX_PROMPTS))
        if w.shape[0] != B or w.shape[2] not in (1, D) or w.shape[3] not in (1, T):
            raise ValueError("y['prompt_weight'] %s must be [%d, K, %d or 1, %d or 1]" % (tuple(w.shape), B, D, T))
        if not bool(torch.isfinite(w).all()):
            raise ValueError("y['prompt_weight'] must be finite")
        w = w.to(torch.float32)
        if self.model.cond_mode == "action":
            a = y.get("prompt_action")
            if a is None:
                raise ValueError("an action model needs y['prompt_action'] [B, K]")
            a = np.asarray(a.detach().cpu() if torch.is_tensor(a) else a)
            if a.shape != (B, K) or not np.issubdtype(a.dtype, np.integer):
                raise ValueError("y['prompt_action'] %s must be integer [%d, %d]" % (a.shape, B, K))
            if ((a < 0) | (a >= int(self.model.num_actions))).any():
                raise ValueError("y['prompt_action'] holds an action outside 0 .. %d" % (int(self.model.num_actions) - 1))
            return None, a.astype(np.int64), w
        e = y.get("prompt_embed")
        if e is None:
            texts = y.get("prompt_text")
            if texts is None:
                raise ValueError("a text model needs y['prompt_embed'] [K, B, C] or y['prompt_text'] (B lists of K strings)")
            if len(texts) != B or any(isinstance(p, str) or len(p) != K for p in texts):
                raise ValueError("y['prompt_text'] must hold B = %d lists of K = %d strings" % (B, K))
            return None, None, w
        C = int(self.model.clip_dim)
        if self.model.text_encoder_type == "bert":
            return _token_prompts(e, K, B, C), None, w
        if not torch.is_tensor(e) or not e.is_floating_point() or tuple(e.shape) != (K, B, C):
            raise ValueError("y['prompt_embed'] must be a float tensor [%d, %d, %d]" % (K, B, C))
        return e, None, w

    def encode_prompts(self, texts):
        """[K, B, C] text features of y['prompt_text'] (B lists of K strings), the model's encode_text per prompt; for the
        BERT decoder the list of K (tokens, mask) pairs."""
        K = len(texts[0])
        enc = [self.model.encode_text([p[k] for p in texts]) for k in range(K)]
        return enc if self.model.text_encoder_type == "bert" else torch.cat(enc, dim=0)

    def forward(self, x, timesteps, y=None):
        self.prompts(y if y is not None else {}, x.shape)       # y's prompts checked before any engine work
        return _run_model(self.model, x, timesteps, y, wrapper=self)


def _token_prompts(e, K, B, C):
    """y['prompt_embed'] of the BERT decoder, checked: a list of K (tokens float [Mt_k, B, C], padding mask bool or
    integer [B, Mt_k]) pairs, 1 <= Mt_k <= MAX_MEMORY_TOKENS."""
    from .. import _lib
    if not isinstance(e, (list, tuple)) or len(e) != K or any(not isinstance(p, tuple) or len(p) != 2 for p in e):
        raise ValueError("the BERT decoder's y['prompt_embed'] must be a list of K = %d (tokens [Mt, %d, %d], mask [%d, Mt]) "
                         "pairs" % (K, B, C, B))
    for k, (tok, msk) in enumerate(e):
        if not torch.is_tensor(tok) or not tok.is_floating_point() or tok.dim() != 3 or tuple(tok.shape[1:]) != (B, C):
            raise ValueError("prompt %d: tokens must be a float tensor [Mt, %d, %d]" % (k, B, C))
        Mt = int(tok.shape[0])
        if not 1 <= Mt <= _lib.MAX_MEMORY_TOKENS:
            raise ValueError("prompt %d: %d tokens outside 1 .. %d" % (k, Mt, _lib.MAX_MEMORY_TOKENS))
        if not torch.is_tensor(msk) or msk.is_floating_point() or msk.is_complex() or tuple(msk.shape) != (B, Mt):
            raise ValueError("prompt %d: the padding mask must be a bool or integer tensor [%d, %d]" % (k, B, Mt))
    return list(e)


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


# A transition is sampled as a sequence of its own: one conditioning token + Lt frames within the engine's 256 keys.
MAX_TRANSITION_FRAMES = 255


def transition_layout(batch, nframes, handshake_size, blend_len, lengths=None, motion_start=None,
                      max_frames=MAX_TRANSITION_FRAMES):
    """Host-only layout of the refined transitions between chained windows (DoubleTake's second take; DESIGN.md,
    "Refined transitions").  For every window b that continues p = b - 1 there is one transition of Lt = 2m + h frames
    (h = handshake_size, m = blend_len): p's last m frames before the handshake, p's copy of the handshake, then b's frames
    h .. h + m - 1.  Returns a dict of numpy arrays:
      pairs [n, 2] (p, b);  src_window, src_frame [n, Lt] where each transition frame comes from in the window batch;
      weight fp32 [Lt] (1 = keep the first take: (m - f)/m, 0 over the handshake, (f - m - h + 1)/m; fp64, rounded once);
      motion [n] the stitched motion (stitch_handshake) each transition belongs to, and paste [n, 2] the frames
      [s - m + 1, s + h + m - 1) of that motion its frames 1 .. Lt - 2 replace, s = where b's handshake begins in it.
    ValueError as handshake_layout raises it, and for m < 1, a chained window with n < h + m, a window chained on both
    sides with n < 2h + 2m (its transitions would overlap), or Lt > max_frames."""
    h, m = int(handshake_size), int(blend_len)
    if m < 1:
        raise ValueError("blend_len must be >= 1 (got %d)" % m)
    n, ms = handshake_layout(batch, nframes, h, lengths, motion_start)
    Lt = 2 * m + h
    chained_prev = ~ms
    chained_next = np.append(~ms[1:], False)
    for b in range(batch):
        if (chained_prev[b] or chained_next[b]) and n[b] < h + m:
            raise ValueError("window %d is chained but has %d frames < handshake_size + blend_len = %d" % (b, n[b], h + m))
        if chained_prev[b] and chained_next[b] and n[b] < 2 * h + 2 * m:
            raise ValueError("window %d has %d frames < 2 x (handshake_size + blend_len) = %d: its two transitions would "
                             "overlap" % (b, n[b], 2 * h + 2 * m))
    if any(chained_prev) and Lt > max_frames:
        raise ValueError("a transition of 2 x blend_len + handshake_size = %d frames exceeds the model's %d" % (Lt, max_frames))
    f = np.arange(Lt)
    w = np.zeros(Lt, dtype=np.float64)
    w[:m] = (m - f[:m]) / m
    w[m + h:] = (f[m + h:] - m - h + 1) / m
    pairs, src_w, src_f, motion, paste = [], [], [], [], []
    k, off = -1, np.zeros(batch, dtype=np.int64)               # off[b]: where window b's frame 0 lies in its motion
    for b in range(batch):
        if ms[b]:
            k += 1
            continue
        p = b - 1
        off[b] = off[p] + n[p] - h
        pairs.append((p, b))
        src_w.append(np.where(f < m + h, p, b))
        src_f.append(np.where(f < m + h, n[p] - h - m + f, f - m))
        motion.append(k)
        paste.append((off[b] - m + 1, off[b] + h + m - 1))
    shape = (len(pairs), Lt)
    return dict(pairs=np.asarray(pairs, dtype=np.int64).reshape(-1, 2),
                src_window=np.asarray(src_w, dtype=np.int64).reshape(shape),
                src_frame=np.asarray(src_f, dtype=np.int64).reshape(shape), weight=w.astype(np.float32),
                motion=np.asarray(motion, dtype=np.int64), paste=np.asarray(paste, dtype=np.int64).reshape(-1, 2))


# per-window entries of y that a transition takes from its later window; flags that hold for the whole batch
_PER_WINDOW_KEYS = ("text_embed", "text", "action", "scale", "target_cond", "target_joint_names", "is_heading")
_BATCH_FLAGS = ("uncond", "target_uncond")


def _transition_y(y, windows, Lt, device):
    """The conditioning of each transition: window b's entries of y (windows = the b of every transition), every one of
    the Lt frames valid.  The window batch's inpainting, lengths, mask and motion_start stay behind."""
    idx = torch.as_tensor(windows, dtype=torch.long)
    out = {k: y[k] for k in _BATCH_FLAGS if k in y}
    for k in _PER_WINDOW_KEYS:
        if k not in y:
            continue
        v = y[k]
        if k == "text_embed" and torch.is_tensor(v):
            out[k] = v if v.shape[1] == 1 else v[:, idx.to(v.device)]          # [1, B, C]; a single prompt is shared
        elif k == "text_embed" and isinstance(v, tuple):                      # BERT: (tokens [Mt, B, C], mask [B, Mt])
            tok, msk = v
            out[k] = (tok if tok.shape[1] == 1 else tok[:, idx.to(tok.device)],
                      msk if msk.shape[0] == 1 else msk[idx.to(msk.device)])
        elif torch.is_tensor(v):
            out[k] = v[idx.to(v.device)]
        elif isinstance(v, np.ndarray):
            out[k] = v[idx.numpy()]
        else:
            out[k] = [v[int(b)] for b in windows]
    n = len(windows)
    out["mask"] = torch.ones((n, 1, 1, Lt), dtype=torch.bool, device=device)
    out["lengths"] = torch.full((n,), Lt, dtype=torch.long, device=device)
    return out


def refine_transitions(sample_fn, model, windows, model_kwargs, handshake_size, blend_len, skip_timesteps,
                       transition_kwargs=None, **sample_kw):
    """DoubleTake's second take (Shafir et al., "Human Motion Diffusion as a Generative Prior"; this project's definition,
    DESIGN.md "Refined transitions"): the motions of a batch of first-take windows (HandshakeSampleModel; laid out by
    model_kwargs['y']['lengths'] / ['motion_start']) with every transition re-noised to depth skip_timesteps and denoised
    again as a short motion of its own, its margins softly pinned to the first take.

    All transitions run as ONE call sample_fn(model, (n, J, F, Lt), skip_timesteps=skip_timesteps, init_image=x_init,
    model_kwargs={'y': y_t}, **sample_kw), y_t carrying y['inpainting_weight'] (transition_layout's weights over J and F)
    and y['inpainted_motion'] = x_init, and by default each transition window b's conditioning (transition_kwargs replaces
    it).  The refined frames 1 .. Lt - 2 are pasted into stitch_handshake's motions; without a chained pair those are
    returned as they are, with no engine call.  `model` is the plain (guided) model: a HandshakeSampleModel raises
    TypeError, a prefix-completion (DiP, context_len > 0) model NotImplementedError; layout errors raise ValueError (transition_layout),
    as does skip_timesteps outside [0, num_timesteps).  Gather and paste are device indexing only."""
    r = resolve(model)
    if r.kind == "joint":
        raise TypeError("refine_transitions is not implemented with joint-position control (JointControlSampleModel)")
    if r.kind == "multi":
        raise TypeError("refine_transitions is not implemented with multi-prompt guidance (MultiPromptSampleModel)")
    if r.kind == "handshake":
        raise TypeError("refine_transitions runs the plain model: pass the model a HandshakeSampleModel wraps, not the wrapper")
    if r.mdm is None:
        raise TypeError("HandshakeSampleModel wraps a b200mdm MDM or ClassifierFreeSampleModel (got %r)" % type(r.core))
    if r.mdm.is_prefix_comp:
        raise NotImplementedError("transitions are not implemented for prefix-completion (DiP) models")
    k = int(skip_timesteps)
    n_steps = getattr(getattr(sample_fn, "__self__", None), "num_timesteps", None)
    if k < 0 or (n_steps is not None and k >= n_steps):
        raise ValueError("skip_timesteps must lie in [0, %s) (got %d)" % (n_steps, k))
    y = model_kwargs["y"]
    B, J, F, T = (int(s) for s in windows.shape)
    h = int(handshake_size)
    lay = transition_layout(B, T, h, blend_len, y.get("lengths"), y.get("motion_start"),
                            min(MAX_TRANSITION_FRAMES, int(r.mdm.pos_embed_max_len) - 1))
    motions = stitch_handshake(windows, y.get("lengths"), h, y.get("motion_start"))
    n = lay["pairs"].shape[0]
    if n == 0:
        return motions
    Lt, dev = lay["weight"].shape[0], windows.device
    sw = torch.from_numpy(lay["src_window"]).to(dev)
    sf = torch.from_numpy(lay["src_frame"]).to(dev)
    x_init = windows[sw, :, :, sf].permute(0, 2, 3, 1).contiguous()          # [n, Lt, J, F] -> [n, J, F, Lt]
    w = torch.from_numpy(lay["weight"]).to(dev).view(1, 1, 1, Lt).expand(n, J, F, Lt).contiguous()
    if transition_kwargs is None:
        kw = {"y": _transition_y(y, lay["pairs"][:, 1], Lt, dev)}
    else:
        kw = dict(transition_kwargs, y=dict(transition_kwargs["y"]))
    kw["y"]["inpainting_weight"] = w
    kw["y"]["inpainted_motion"] = x_init
    refined = sample_fn(model, (n, J, F, Lt), skip_timesteps=k, init_image=x_init, model_kwargs=kw, **sample_kw)
    for i in range(n):
        a, b = (int(v) for v in lay["paste"][i])
        motions[int(lay["motion"][i])][..., a:b] = refined[i, ..., 1:Lt - 1]
    return motions


# the samplers whose chain runs as engine loops (GaussianDiffusion._ar_chain), and the keywords each takes there; every
# other keyword of theirs must keep its default (hooks, init_image / skip_timesteps, dump_steps, const_noise, noise_fn)
_CHAIN_SAMPLERS = {"p_sample_loop": "MODE_DDPM", "ddim_sample_loop": "MODE_DDIM", "dpm_solver_sample_loop": "MODE_DPM"}
_CHAIN_KEYS = {"model_kwargs", "noise", "clip_denoised", "device", "progress", "use_graph", "noise_seed",
               "sample_index_base", "noise_tape", "eta", "order"}
_CHAIN_DEFAULTS = dict(denoised_fn=None, cond_fn=None, skip_timesteps=0, init_image=None, randomize_class=False,
                       cond_fn_with_grad=False, dump_steps=None, const_noise=False, noise_fn=None)


def _chain_plan(sample_fn, model, ar_shape, n_chunks, kargs):
    """(diffusion, mode, keywords of GaussianDiffusion._ar_chain) when AutoRegressiveSampler.sample's chain gives the
    same result as engine loops, else None (the host chain runs): sample_fn is p_sample_loop, ddim_sample_loop or
    dpm_solver_sample_loop (order 1 or 2) of a b200mdm GaussianDiffusion / SpacedDiffusion, as its class defines it; the
    model a DiP MDM or its ClassifierFreeSampleModel; no keyword outside _CHAIN_KEYS unless at its default; a noise_tape
    only for DDPM / DDIM, without noise_seed, and every tape and x_T of the chain's shapes; a float32 y['prefix']."""
    from ..diffusion import gaussian_diffusion as gd
    from .. import _lib
    diffusion, func = getattr(sample_fn, "__self__", None), getattr(sample_fn, "__func__", None)
    if not isinstance(diffusion, gd.GaussianDiffusion):
        return None
    name = next((k for k in _CHAIN_SAMPLERS if func is getattr(gd.GaussianDiffusion, k)), None)
    if name is None:
        return None
    core = _core(model)
    if core is None or not (core[0].is_prefix_comp and core[0].is_dip):
        return None
    def at_default(k):
        v, d = kargs[k], _CHAIN_DEFAULTS[k]
        return v is None if d is None else (isinstance(v, (bool, int, np.integer)) and v == d)
    if any(k not in _CHAIN_KEYS and (k not in _CHAIN_DEFAULTS or not at_default(k)) for k in kargs):
        return None
    if "noise_fn" in kargs and name != "p_sample_loop":          # the other two have no such keyword (TypeError)
        return None
    mode = getattr(_lib, _CHAIN_SAMPLERS[name])
    kw = {k: kargs[k] for k in _CHAIN_KEYS - {"model_kwargs", "progress", "eta", "order"} if k in kargs}
    if name == "ddim_sample_loop":
        kw["eta"] = kargs.get("eta", 0.0)
    elif "eta" in kargs:
        return None
    if name == "dpm_solver_sample_loop":
        order = kargs.get("order", 2)
        if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or order not in (1, 2):
            return None
        if kw.get("noise_tape") is not None:
            return None
        kw["order"] = int(order)
    elif "order" in kargs:
        return None
    tape, noise = kw.get("noise_tape"), kw.get("noise")
    shape = tuple(ar_shape)
    if tape is not None and (kw.get("noise_seed") is not None or not torch.is_tensor(tape) or tape.dim() != len(shape) + 2
                             or tape.shape[0] < n_chunks or tape.shape[1] != diffusion.num_timesteps
                             or tuple(tape.shape[2:]) != shape):
        return None
    if noise is not None and not (torch.is_tensor(noise) and (tuple(noise.shape) == shape or (
            noise.dim() == len(shape) + 1 and noise.shape[0] >= n_chunks and tuple(noise.shape[1:]) == shape))):
        return None
    y = (kargs.get("model_kwargs") or {}).get("y")
    if not isinstance(y, dict) or not torch.is_tensor(y.get("prefix")) or y["prefix"].dtype != torch.float32:
        return None
    return diffusion, mode, kw


class AutoRegressiveSampler:
    """DiP's outer loop (reference utils/sampler_util.py:41-81): generate `required_frames` as a chain of `pred_len`
    chunks, each a full diffusion loop of the trans_dec engine conditioned on the last `context_len` frames of the
    previous chunk (y['prefix']).  With p_sample_loop, ddim_sample_loop or dpm_solver_sample_loop of a b200mdm diffusion
    (_chain_plan), the whole chain runs as engine loops: the conditioning is set once, and the prefix hand-off between
    chunks happens on the device, with the same result bit for bit (DESIGN.md, "Autoregressive chain").  Any other
    sample_fn runs here on the host, one `sample_fn` call per chunk.  The caller's kwargs are never mutated (the
    reference deep-copies them per chunk; here only the dicts that change are rebuilt).

    Goals in the world frame (DESIGN.md, "Goals in the world frame"): y['target_world'] [B, n_ext, 3] (one goal for the
    whole chain) or [n_chunks, B, n_ext, 3] (a waypoint per chunk), in target_cond's layout and validity keys, is
    re-expressed in each chunk's own frame on the device and given to that chunk as its target; mean / std [D] are the
    dataset normalisation that recover_from_ric needs.  W is the frame of recover_from_ric on the returned motion."""

    def __init__(self, args, sample_fn, required_frames=196, *, mean=None, std=None):
        self.sample_fn = sample_fn
        self.args = args
        self.required_frames = required_frames
        self.mean, self.std = mean, std

    def _goal(self, model, y, batch, n_chunks):
        """(goals [n_goals, B, n_ext, 3] fp32, validity uint8 [B, n_ext]) of y['target_world'], or None without it or
        with y['target_uncond']; ValueError for keys that clash, before any engine work."""
        if "target_world" not in y:
            return None
        if "target_cond" in y:
            raise ValueError("y['target_world'] and y['target_cond'] both give the target: pass one of them")
        mdm = resolve(model).mdm
        if mdm is None or not mdm.multi_target_cond:
            raise ValueError("y['target_world'] was given, but the model has no target encoder (multi_target_cond=False)")
        if self.mean is None or self.std is None:
            raise ValueError("y['target_world'] needs AutoRegressiveSampler(..., mean=, std=), the dataset normalisation")
        g = y["target_world"]
        if not torch.is_tensor(g):
            g = torch.as_tensor(np.asarray(g, dtype=np.float32))
        n_ext = len(mdm.extended_goal_joint_names)
        if g.dim() == 3:
            g = g[None]
        elif g.dim() != 4 or g.shape[0] != n_chunks:
            raise ValueError("y['target_world'] must be [B, %d, 3] or [n_chunks = %d, B, %d, 3] (got %s)"
                             % (n_ext, n_chunks, n_ext, tuple(g.shape)))
        for v, name in ((self.mean, "mean"), (self.std, "std")):
            if tuple(v.shape) != (mdm.njoints * mdm.nfeats,):
                raise ValueError("%s must be [%d] (got %s)" % (name, mdm.njoints * mdm.nfeats, tuple(v.shape)))
        from ..engine import canonical_target
        _, valid = canonical_target(dict(y, target_cond=g[0]), batch, mdm.extended_goal_joint_names)
        if bool(y.get("target_uncond", False)):
            return None
        return g.to(torch.float32), valid

    def sample(self, model, shape, **kargs):
        if resolve(model).kind == "joint":
            raise NotImplementedError("the autoregressive chain is not implemented with joint-position control")
        pred_len, context_len = self.args.pred_len, self.args.context_len
        n_iterations = self.required_frames // pred_len + int(self.required_frames % pred_len > 0)
        y0 = kargs["model_kwargs"]["y"]
        goal = self._goal(model, y0, shape[0], n_iterations)
        if "target_world" in y0:
            y0 = {k: v for k, v in y0.items() if k != "target_world"}
        cur_prefix = y0["prefix"].clone()
        dynamic_text_mode = isinstance(y0["text"][0], list) if "text" in y0 else False   # a prompt per chunk
        samples_buf = [cur_prefix] if getattr(self.args, "autoregressive_include_prefix", False) else []
        ar_shape = list(shape)
        ar_shape[-1] = pred_len
        tape = kargs.get("noise_tape")            # b200mdm extension: one tape per chunk, [n_iterations, n_run+1, ...]
        plan = _chain_plan(self.sample_fn, model, ar_shape, n_iterations, kargs)
        if plan is not None:
            ys = []
            for i in range(n_iterations):
                y = dict(y0)
                if dynamic_text_mode:
                    y["text"] = [s[i] for s in y0["text"]]
                    if getattr(model, "text_encoder_type", "bert") != "bert":
                        raise NotImplementedError("DiP model only supports BERT text encoder at the moment.")
                    y["text_embed"] = (y0["text_embed"][0][:, :, i], y0["text_embed"][1][:, i])
                ys.append(y)
            diffusion, mode, kw = plan
            if goal is not None:
                kw = dict(kw, goal=(self.mean, self.std) + goal)
            out = diffusion._ar_chain(mode, model, ar_shape, ys, self.required_frames, bool(samples_buf), **kw)
            if out is not None:
                return out
        if goal is not None:            # the carry stays on the device; each chunk's target is computed there
            from ..engine import Engine
            dev = next(model.parameters()).device
            g, mean, std = (t.to(dev) for t in (goal[0], self.mean, self.std))
            carry = torch.zeros(shape[0], 6, dtype=torch.float64, device=dev)
            first = cur_prefix if samples_buf else cur_prefix[..., :0]
            target = Engine.chunk_frame(carry, first.to(dev), mean, std, g[0])
        for i in range(n_iterations):
            y = dict(y0)
            y["prefix"] = cur_prefix
            if goal is not None:
                y["target_cond"] = target
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
            if goal is not None and i + 1 < n_iterations:
                target = Engine.chunk_frame(carry, samples_buf[-1].to(dev), mean, std, g[min(i + 1, g.shape[0] - 1)])
        return torch.cat(samples_buf, dim=-1)[..., :self.required_frames]
