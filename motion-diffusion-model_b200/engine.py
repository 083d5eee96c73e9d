"""Thin Python wrapper over the C ABI (include/b200mdm.h): torch tensors in, torch tensors out.

Everything numeric happens inside libb200mdm.so; this module only marshals pointers, keeps the tensors that
the engine references alive, and canonicalises the reference's untyped ``y`` dict into the POD arguments of
``b200mdm_set_cond``.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import check


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def canonical_target(y, batch, joint_names):
    """(target [B, n_ext, 3] fp32 tensor, validity uint8 [B, n_ext] numpy) from the reference's y keys: validity is 1
    for each joint named in y['target_joint_names'][b], plus 'heading' when y['is_heading'][b] (model/mdm.py:410-416).
    An unknown joint name raises ValueError (the reference's list.index)."""
    tc = y["target_cond"]
    if not torch.is_tensor(tc):
        tc = torch.as_tensor(np.asarray(tc, dtype=np.float32))
    n = len(joint_names)
    if tuple(tc.shape) != (batch, n, 3):
        raise ValueError("y['target_cond'] must be [batch, %d, 3] (got %s)" % (n, tuple(tc.shape)))
    names, heading = y.get("target_joint_names"), y.get("is_heading")
    if names is None or heading is None:
        raise ValueError("y['target_cond'] needs y['target_joint_names'] and y['is_heading']")
    if torch.is_tensor(heading):
        heading = heading.detach().cpu().numpy()
    heading = np.asarray(heading).reshape(-1)
    if len(names) != batch or heading.shape[0] != batch:
        raise ValueError("y['target_joint_names'] and y['is_heading'] need one entry per sample")
    valid = np.zeros((batch, n), dtype=np.uint8)
    for b in range(batch):
        sample = [str(j) for j in np.asarray(names[b], dtype=object).reshape(-1)]
        if heading[b]:
            sample.append("heading")
        for j in sample:
            if j not in joint_names:
                raise ValueError("unknown target joint %r (known: %s)" % (j, ", ".join(joint_names)))
            valid[b, joint_names.index(j)] = 1
    return tc, valid


def _lengths_host(lengths, B):
    """y['lengths'] (tensor, array or None) -> contiguous int64 numpy [B], or None"""
    if lengths is None:
        return None
    n = np.ascontiguousarray(np.asarray(lengths.detach().cpu() if torch.is_tensor(lengths) else lengths, dtype=np.int64).reshape(-1))
    assert n.shape == (B,), n.shape
    return n


def _grid(grid, device):
    """(b200mdm_grid, the fp32 values on `device` it points to) of a SceneGrid, or (None, None)"""
    if grid is None:
        return None, None
    v = grid.values.to(device=device, dtype=torch.float32).contiguous()
    gz, gx = grid.shape
    return _lib.Grid(v.data_ptr(), gz * gx if grid.per_sample else 0, gz, gx, grid.origin[0], grid.origin[1], grid.cell), v


def _grid_ref(g):
    return None if g is None else ctypes.byref(g)


def _interaction(characters, weight, margin, placement, pairs, reach, pair_weight, device):
    """(the interaction arguments of b200mdm_set_interaction_guidance after the engine, the tensors they point to):
    placement [B, 3], pairs int [N, 4] or None, reach [N], pair_weight [N, T] (every scene) or [B / C, N, T]"""
    pl = placement.to(device=device, dtype=torch.float32).contiguous()
    n = 0 if pairs is None else int(pairs.shape[0])
    if n == 0:
        return (int(characters), float(weight), float(margin), _ptr(pl), None, 0, None, None, 0), (pl,)
    rows = np.ascontiguousarray(np.asarray(pairs.cpu() if torch.is_tensor(pairs) else pairs, dtype=np.int32).reshape(n, 4))
    dist = np.ascontiguousarray(np.asarray(reach.cpu() if torch.is_tensor(reach) else reach, dtype=np.float32).reshape(n))
    pw = pair_weight.to(device=device, dtype=torch.float32).contiguous()
    stride = int(pw.shape[1] * pw.shape[2]) if pw.dim() == 3 else 0
    return ((int(characters), float(weight), float(margin), _ptr(pl), rows.ctypes.data_as(ctypes.c_void_p), n,
             dist.ctypes.data_as(ctypes.c_void_p), _ptr(pw), stride), (pl, rows, dist, pw))


def _guidance_hook(fn, x0, mean, std, target, weight, step, iters, foot=(), scene=(), interaction=()):
    """The guidance iterations of the test hook `fn` (b200mdm_test_*_guidance) on x0's device: (guided x0 [B, D, T],
    total G [iters + 1, B]).  foot: (contact_weight, floor_weight, floor_height, contact, lengths); scene:
    (obstacle_weight, obstacle_margin, sdf, terrain); interaction: the arguments of _interaction before the device."""
    lib = _lib.load()
    x0, mean, std, target, weight = (t.to(torch.float32).contiguous() for t in (x0, mean, std, target, weight))
    B, D, T = int(x0.shape[0]), int(x0.shape[1]), int(x0.shape[-1])
    head, tail = [], []                    # the arguments before B and after iters (locals keep what they point to)
    if foot:
        contact_weight, floor_weight, floor_height, contact, lengths = foot
        kappa = None if contact is None else contact.to(device=x0.device, dtype=torch.float32).contiguous()
        n = _lengths_host(lengths, B)
        head = [_ptr(kappa), None if n is None else n.ctypes.data_as(ctypes.c_void_p)]
        tail += [float(contact_weight), float(floor_weight), float(floor_height)]
    if scene:
        obstacle_weight, obstacle_margin, sdf, terrain = scene
        (gs, vs), (gt, vt) = _grid(sdf, x0.device), _grid(terrain, x0.device)
        tail += [float(obstacle_weight), float(obstacle_margin), _grid_ref(gs), _grid_ref(gt)]
    if interaction:
        args, keep = _interaction(*interaction, x0.device)
        tail += list(args)
    out = torch.empty_like(x0)
    loss = torch.empty((int(iters) + 1, B), device=x0.device, dtype=torch.float32)
    check(getattr(lib, fn)(_ptr(x0), _ptr(mean), _ptr(std), _ptr(target), _ptr(weight), *head, B, T, D, float(step),
                           int(iters), *tail, _ptr(out), _ptr(loss), _stream()))
    return out, loss


def joint_guidance_hook(x0, mean, std, target, weight, step, iters):
    """The guidance iterations of joint-position control alone (b200mdm_test_joint_guidance), on x0's device:
    (guided x0 [B, D, T], loss [iters + 1, B])."""
    return _guidance_hook("b200mdm_test_joint_guidance", x0, mean, std, target, weight, step, iters)


def foot_guidance_hook(x0, mean, std, target, weight, step, iters, contact_weight, floor_weight, floor_height=0.0,
                       contact=None, lengths=None):
    """The guidance iterations with the foot-contact and floor terms alone (b200mdm_test_foot_guidance), on x0's device:
    (guided x0 [B, D, T], total G [iters + 1, B]).  contact [B, 4, T] or None (derived from x0), lengths [B] or None."""
    return _guidance_hook("b200mdm_test_foot_guidance", x0, mean, std, target, weight, step, iters,
                          (contact_weight, floor_weight, floor_height, contact, lengths))


def scene_guidance_hook(x0, mean, std, target, weight, step, iters, contact_weight, floor_weight, floor_height,
                        obstacle_weight, obstacle_margin, sdf=None, terrain=None, contact=None, lengths=None):
    """The guidance iterations with the foot and scene terms alone (b200mdm_test_scene_guidance), on x0's device:
    (guided x0 [B, D, T], total G [iters + 1, B]).  sdf / terrain: SceneGrid or None; contact, lengths as
    foot_guidance_hook's."""
    return _guidance_hook("b200mdm_test_scene_guidance", x0, mean, std, target, weight, step, iters,
                          (contact_weight, floor_weight, floor_height, contact, lengths),
                          (obstacle_weight, obstacle_margin, sdf, terrain))


def interaction_guidance_hook(x0, mean, std, target, weight, step, iters, contact_weight, floor_weight, floor_height,
                              obstacle_weight, obstacle_margin, sdf, terrain, characters, interaction_weight,
                              interaction_margin, placement, pairs=None, reach=None, pair_weight=None, contact=None,
                              lengths=None):
    """The guidance iterations with the foot, scene and interaction terms alone (b200mdm_test_interaction_guidance), on
    x0's device: (guided x0 [B, D, T], total G [iters + 1, B], each pair's energy at its lower rank).  placement [B, 3],
    pairs int [N, 4] scene-local (a, j, b, k) or None, reach [N], pair_weight [N, T] or [B / C, N, T]; the other
    arguments as scene_guidance_hook's."""
    return _guidance_hook("b200mdm_test_interaction_guidance", x0, mean, std, target, weight, step, iters,
                          (contact_weight, floor_weight, floor_height, contact, lengths),
                          (obstacle_weight, obstacle_margin, sdf, terrain),
                          (characters, interaction_weight, interaction_margin, placement, pairs, reach, pair_weight))


class Engine:
    """One engine per model instance (weights + workspace live on the current CUDA device)."""

    def __init__(self, *, arch, latent_dim, ff_size, num_layers, num_heads, njoints, nfeats, cond_mode, cond_dim,
                 num_actions, mask_frames, pos_embed_max_len, temb_rows, context_len=0, target_encoder=None,
                 target_enc_layers=1, target_joint_names=(), emb_trans_dec=False, dec_memory=_lib.DEC_MEMORY_TOKENS):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("b200mdm needs a CUDA device (sm_90a); there is no CPU fallback")
        cm = _lib.COND_TEXT if "text" in cond_mode else _lib.COND_ACTION if "action" in cond_mode else _lib.COND_NONE
        self.cfg = _lib.Config(arch=_lib.ARCH[arch], latent_dim=latent_dim, ff_size=ff_size, num_layers=num_layers,
                               num_heads=num_heads, njoints=njoints, nfeats=nfeats, cond_mode=cm, cond_dim=cond_dim,
                               num_actions=num_actions, mask_frames=int(bool(mask_frames)),
                               pos_embed_max_len=pos_embed_max_len, temb_rows=temb_rows, context_len=context_len,
                               target_encoder=_lib.TARGET[target_encoder] if target_encoder else 0,
                               target_enc_layers=target_enc_layers if target_encoder else 0,
                               target_joints=len(target_joint_names) if target_encoder else 0,
                               emb_trans_dec=int(bool(emb_trans_dec)), dec_memory=dec_memory)
        self.target_encoder = target_encoder
        self.target_joint_names = list(target_joint_names)     # extended list: goal joints + ['traj', 'heading']
        self.dec = arch == "trans_dec"
        self.dec_clip = self.dec and dec_memory == _lib.DEC_MEMORY_CLIP
        self.context_len = context_len
        h = ctypes.c_void_p()
        check(self.lib.b200mdm_create(ctypes.byref(self.cfg), ctypes.byref(h)))
        self.h = h
        self.cond_mode = cm
        self._keep = {}
        self._cond_key = None
        self._sched_key = None
        self._table_keys = {}                     # "next" / "dpm" / "vb": the key of the rows uploaded for the schedule
        self.batch = self.nframes = self.n_tokens = 0
        self.halves = 1
        self.groups = 0                           # G = K + 1 under multi-prompt guidance, else 0

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200mdm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd):
        for name, t in sd.items():
            if not torch.is_tensor(t):
                continue
            if self.target_encoder == "multi" and name.startswith("embed_target_cond.target_loc_emb."):
                # the C ABI names the multi encoder's per-joint MLP by the joint's index in the extended list
                joint, _, rest = name[len("embed_target_cond.target_loc_emb."):].partition(".")
                if joint in self.target_joint_names:
                    name = "embed_target_cond.target_loc_emb.%d.%s" % (self.target_joint_names.index(joint), rest)
            t = t.detach().to(torch.float32).contiguous()
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            check(self.lib.b200mdm_load_weight(self.h, name.encode(), _ptr(t), shape, t.dim()))
        check(self.lib.b200mdm_finalize_weights(self.h, _stream()))
        self._cond_key = None

    # ------------------------------------------------------------------ schedule
    def set_schedule(self, rows, timestep_map, key=None):
        if key is not None and key == self._sched_key:
            return
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        tmap = np.ascontiguousarray(timestep_map, dtype=np.int32)
        assert rows.shape == (len(tmap), _lib.SCHED_STRIDE)
        check(self.lib.b200mdm_set_schedule(self.h, len(tmap), rows.ctypes.data_as(ctypes.c_void_p),
                                            tmap.ctypes.data_as(ctypes.c_void_p)))
        self._sched_key = key
        self._table_keys.clear()                  # the engine marks the reverse, DPM-Solver++ and bound tables stale

    def _set_table(self, which, rows, key):
        """b200mdm_set_schedule_<which>, skipped when `key` names the rows already uploaded for this schedule."""
        if key is not None and key == self._table_keys.get(which):
            return
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        assert rows.ndim == 2 and rows.shape[1] == getattr(_lib, "SCHED_%s_STRIDE" % which.upper())
        setter = getattr(self.lib, "b200mdm_set_schedule_" + which)
        check(setter(self.h, rows.shape[0], rows.ctypes.data_as(ctypes.c_void_p)))
        self._table_keys[which] = key

    def set_schedule_next(self, rows, key=None):
        """[n_steps, 2] fp32 rows sqrt(abn), sqrt(1 - abn) of the current schedule (b200mdm_set_schedule_next)."""
        self._set_table("next", rows, key)

    def set_schedule_dpm(self, rows, key=None):
        """[n_steps, 4] fp32 rows c_x, c0, c_cur, c_prev of the current schedule (b200mdm_set_schedule_dpm)."""
        self._set_table("dpm", rows, key)

    def set_schedule_vb(self, rows, key=None):
        """[n_steps, 12] fp32 rows of the variational-bound table of the current schedule (b200mdm_set_schedule_vb)."""
        self._set_table("vb", rows, key)

    # ------------------------------------------------------------------ conditioning
    def set_cond(self, batch, nframes, y, guided, device):
        """Canonicalise model_kwargs['y'] (data_loaders/tensors.py:22-64 schema).  `guided` => CFG pair."""
        y = y or {}
        if self.dec:
            self._set_cond_dec(batch, nframes, y, guided, device)
        else:
            self._set_cond_enc(batch, nframes, y, guided, device)
        self._set_target(batch, y, device)

    def _set_target(self, batch, y, device):
        """y['target_cond'] [B, n_ext, 3], y['target_joint_names'] (per sample, a list or array of joint names),
        y['is_heading'] [B] (model/mdm.py:197-199).  Both CFG halves carry the target (the guidance wrapper never sets
        target_uncond, utils/sampler_util.py:27-34); y['target_uncond'] = True samples without it, as does a y without
        'target_cond' (the b200mdm_set_cond* call above has cleared the previous target)."""
        self._keep.pop("target", None)
        if "target_cond" not in y or bool(y.get("target_uncond", False)):
            return
        if not self.target_encoder:
            raise ValueError("y['target_cond'] was given, but the model has no target encoder (multi_target_cond=False)")
        tc, valid = canonical_target(y, batch, self.target_joint_names)
        tc = tc.to(device=device, dtype=torch.float32).contiguous()
        check(self.lib.b200mdm_set_target(self.h, _ptr(tc), valid.ctypes.data_as(ctypes.c_void_p), _stream()))
        self._keep["target"] = tc

    def test_target(self, target, valid):
        """The device target encoder alone (b200mdm_test_target): g [B, d] for target [B, n_ext, 3] (device fp32) and
        valid uint8 [B, n_ext] (numpy)."""
        target = target.to(torch.float32).contiguous()
        valid = np.ascontiguousarray(valid, dtype=np.uint8)
        out = torch.empty(target.shape[0], self.cfg.latent_dim, device=target.device, dtype=torch.float32)
        check(self.lib.b200mdm_test_target(self.h, _ptr(target), valid.ctypes.data_as(ctypes.c_void_p), target.shape[0],
                                           _ptr(out), _stream()))
        return out

    def packed_batch(self):
        """Bp, the rows of the packed batch of the conditioning set last: G * batch under multi-prompt guidance (G = K + 1
        groups), else halves * batch (2 with classifier-free guidance)."""
        return (self.groups or self.halves) * self.batch

    def test_cross_rows(self, timestep, halves=None, device="cuda"):
        """The CLIP decoder's per-step cross-attention rows (b200mdm_test_cross_rows) for the conditioning last set:
        [num_layers, Bp, d] fp32 at model timestep `timestep`, Bp = packed_batch().  `halves`, when given, must describe
        the same rows (halves * batch = Bp; under multi-prompt guidance halves = G): ValueError otherwise."""
        if halves is not None and int(halves) * self.batch != self.packed_batch():
            raise ValueError("halves = %d gives %d rows, but the conditioning set last packs %d"
                             % (int(halves), int(halves) * self.batch, self.packed_batch()))
        out = torch.empty(self.cfg.num_layers, self.packed_batch(), self.cfg.latent_dim, device=device, dtype=torch.float32)
        check(self.lib.b200mdm_test_cross_rows(self.h, int(timestep), _ptr(out), _stream()))
        return out

    def _set_cond_enc(self, batch, nframes, y, guided, device):
        text_embed = y.get("text_embed")
        if isinstance(text_embed, tuple):
            raise NotImplementedError("BERT (tokens, mask) conditioning belongs to the trans_dec path")
        ln, sc = self._lengths_and_scale(batch, y, guided, device)
        uncond = bool(y.get("uncond", False))
        action = y.get("action")
        te = None
        if text_embed is not None and self.cond_mode == _lib.COND_TEXT:
            te = self._text_rows(text_embed, batch, device)
        ac = None
        if action is not None and self.cond_mode == _lib.COND_ACTION:
            ac = np.ascontiguousarray(action.detach().reshape(batch, -1)[:, 0].cpu().numpy().astype(np.int64))
        check(self.lib.b200mdm_set_cond(self.h, batch, nframes, _ptr(te),
                                        None if ln is None else ln.ctypes.data_as(ctypes.c_void_p), _ptr(sc),
                                        int(uncond), None if ac is None else ac.ctypes.data_as(ctypes.c_void_p),
                                        _stream()))
        self._keep["cond"] = (te, sc)
        self.batch, self.nframes, self.halves, self.n_tokens = batch, nframes, 2 if sc is not None else 1, 1
        self.groups = 0

    def _text_rows(self, te, batch, device):
        """y['text_embed'] [1, B, cond_dim] (or [1, 1, cond_dim]: one prompt for the whole batch, sample/predict.py) as
        contiguous fp32 rows [batch, cond_dim] on `device`."""
        te = te.detach().to(device=device, dtype=torch.float32)
        te = te.reshape(-1, te.shape[-1])
        if te.shape[0] == 1 and batch > 1:
            te = te.expand(batch, -1)
        te = te.contiguous()
        assert te.shape == (batch, self.cfg.cond_dim), (te.shape, batch, self.cfg.cond_dim)
        return te

    @staticmethod
    def _lengths_and_scale(batch, y, guided, device):
        """(lengths int64 numpy or None, scale fp32 device tensor or None) from y['lengths'] / y['mask'] / y['scale']:
        no key mask when the mask has one column (model/mdm.py:242), lengths from a prefix mask (tensors.py:3-6)."""
        lengths, mask = y.get("lengths"), y.get("mask")
        if mask is not None and mask.shape[-1] <= 1:
            lengths = None
        elif lengths is None and mask is not None:
            lengths = mask.reshape(mask.shape[0], -1).sum(-1)
        ln = None
        if lengths is not None:
            ln = np.ascontiguousarray(lengths.detach().reshape(-1).cpu().numpy().astype(np.int64))
            assert ln.shape[0] == batch
        scale = y.get("scale") if guided else None
        if guided and scale is None:
            raise AssertionError("ClassifierFreeSampleModel needs y['scale'] (sampler_util.py:34)")
        sc = None
        if scale is not None:
            sc = scale.detach().to(device=device, dtype=torch.float32).reshape(-1).contiguous()
            assert sc.shape[0] == batch
        return ln, sc

    def _set_cond_dec_clip(self, batch, nframes, y, guided, device):
        """trans_dec with emb_trans_dec (humanml-decoder-with-emb): y['text_embed'] = CLIP features [1, B, 512] (or
        [1, 1, 512] for the whole batch) is the one memory token of each sample (model/mdm.py:218-220,262-264)."""
        te = y.get("text_embed")
        if isinstance(te, tuple):
            raise NotImplementedError("BERT (tokens, mask) conditioning belongs to the DiP decoder (text_encoder_type='bert')")
        uncond = bool(y.get("uncond", False))
        if te is None and uncond and not guided:              # mask_cond zeroes the features (model/mdm.py:218)
            te = torch.zeros(batch, self.cfg.cond_dim, device=device)
        if te is None:
            raise RuntimeError("the CLIP decoder needs y['text_embed'] [1, B, %d] (or y['text'] with a text encoder "
                               "attached)" % self.cfg.cond_dim)
        te = self._text_rows(te, batch, device)
        ln, sc = self._lengths_and_scale(batch, y, guided, device)
        no_pad = np.zeros((batch, 1), dtype=np.uint8)           # the reference passes no memory mask
        check(self.lib.b200mdm_set_cond_dec(self.h, batch, nframes, _ptr(te), no_pad.ctypes.data_as(ctypes.c_void_p), 1,
                                            None if ln is None else ln.ctypes.data_as(ctypes.c_void_p), _ptr(sc),
                                            int(uncond), _stream()))
        self._keep["cond"] = (te, sc)
        self.batch, self.nframes, self.halves, self.n_tokens = batch, nframes, 2 if sc is not None else 1, 1
        self.groups = 0

    def dec_memory(self, te, batch, device):
        """(tokens [Mt, batch, cond_dim] contiguous fp32 on device, padding mask uint8 numpy [batch, Mt]) of a DiP
        y['text_embed'] = (tokens, mask), a single prompt's [Mt, 1, C] / [1, Mt] broadcast over the batch."""
        enc, tmask = te
        enc = enc.detach().to(device=device, dtype=torch.float32)
        if enc.shape[1] == 1 and batch > 1:
            enc = enc.expand(-1, batch, -1)
        enc = enc.contiguous()
        if tmask.shape[0] == 1 and batch > 1:                  # model/mdm.py:215-216
            tmask = torch.repeat_interleave(tmask, batch, dim=0)
        Mt = enc.shape[0]
        assert enc.shape == (Mt, batch, self.cfg.cond_dim) and tuple(tmask.shape) == (batch, Mt), (enc.shape, tmask.shape)
        return enc, np.ascontiguousarray(tmask.detach().cpu().numpy().astype(np.uint8))

    def _set_cond_dec(self, batch, nframes, y, guided, device):
        """DiP: y['text_embed'] = (BERT tokens [Mt,B,768], padding mask [B,Mt] True = pad), y['prefix'] [B,J,F,ctx]
        (reference model/mdm.py:203-206,210-217,264)."""
        if self.dec_clip:
            return self._set_cond_dec_clip(batch, nframes, y, guided, device)
        te = y.get("text_embed")
        if not isinstance(te, tuple):
            raise RuntimeError("trans_dec (DiP) needs y['text_embed'] = (tokens, mask) from bert_encode_text "
                               "(model/mdm.py:180-187)")
        enc, tm = self.dec_memory(te, batch, device)
        Mt = enc.shape[0]
        ln, sc = self._lengths_and_scale(batch, y, guided, device)
        check(self.lib.b200mdm_set_cond_dec(self.h, batch, nframes, _ptr(enc), tm.ctypes.data_as(ctypes.c_void_p), Mt,
                                            None if ln is None else ln.ctypes.data_as(ctypes.c_void_p), _ptr(sc),
                                            int(bool(y.get("uncond", False))), _stream()))
        pf = None
        if self.context_len > 0:
            if "prefix" not in y:
                raise KeyError("prefix completion needs y['prefix'] [B, njoints, nfeats, context_len] (model/mdm.py:204)")
            pf = y["prefix"].detach().to(device=device, dtype=torch.float32).contiguous()
            assert tuple(pf.shape) == (batch, self.cfg.njoints, self.cfg.nfeats, self.context_len), pf.shape
            check(self.lib.b200mdm_set_prefix(self.h, _ptr(pf), _stream()))
        self._keep["cond"] = (enc, sc, pf)
        self.batch, self.nframes, self.halves, self.n_tokens = batch, nframes, 2 if sc is not None else 1, Mt
        self.groups = 0

    def prompt_memories(self, pairs, batch, device):
        """(tokens fp32 [K, Mt, batch, C] contiguous on device, padding mask uint8 numpy [K, batch, Mt]) of K BERT
        (tokens [Mt_k, batch, C], mask [batch, Mt_k]) pairs, each padded to the longest Mt with masked zero tokens."""
        Mt = max(int(t.shape[0]) for t, _ in pairs)
        tok = torch.zeros(len(pairs), Mt, batch, self.cfg.cond_dim, device=device, dtype=torch.float32)
        mask = np.ones((len(pairs), batch, Mt), dtype=np.uint8)
        for k, (t, m) in enumerate(pairs):
            tok[k, :t.shape[0]] = t.detach().to(device=device, dtype=torch.float32)
            mask[k, :, :t.shape[0]] = m.detach().cpu().numpy() != 0
        return tok, mask

    def set_inpaint(self, mask, motion):
        if mask is None:
            check(self.lib.b200mdm_set_inpaint(self.h, None, None))
            self._keep.pop("inpaint", None)
            return
        m8 = mask.to(torch.uint8).contiguous()
        mo = motion.to(torch.float32).contiguous()
        check(self.lib.b200mdm_set_inpaint(self.h, _ptr(m8), _ptr(mo)))
        self._keep["inpaint"] = (m8, mo)

    def set_inpaint_weight(self, weight, motion):
        """Soft inpainting (b200mdm_set_inpaint_weight): weight and motion [B, J, F, T], on the engine's device.  It
        replaces a bool mask; the values are checked by the sampler (gaussian_diffusion._inpainting)."""
        w = weight.to(torch.float32).contiguous()
        mo = motion.to(torch.float32).contiguous()
        check(self.lib.b200mdm_set_inpaint_weight(self.h, _ptr(w), _ptr(mo)))
        self._keep["inpaint"] = (w, mo)

    def set_handshake(self, handshake_size, batch, nframes, y):
        """Handshakes between the chained windows of the batch (b200mdm_set_handshake) from y['lengths'] and
        y['motion_start']; after set_cond, which clears them.  ValueError (before the engine is touched) as
        utils/sampler_util.handshake_layout raises it."""
        from .utils.sampler_util import handshake_layout
        y = y or {}
        n, ms = handshake_layout(batch, nframes, handshake_size, y.get("lengths"), y.get("motion_start"))
        n, ms = np.ascontiguousarray(n), np.ascontiguousarray(ms.astype(np.uint8))
        check(self.lib.b200mdm_set_handshake(self.h, int(handshake_size), n.ctypes.data_as(ctypes.c_void_p),
                                             ms.ctypes.data_as(ctypes.c_void_p), _stream()))

    def _keep_guide(self, term, tensors):
        """keep the tensors of guidance term `term` (0 joint, 1 foot, 2 scene, 3 interaction) alive, and drop those of
        the terms above it, which its setter cleared"""
        self._keep["guide"] = (self._keep.get("guide", []) + [None] * term)[:term] + [tensors]

    def set_joint_guidance(self, mean, std, target, weight, step, iters):
        """Joint-position control for the next DDPM / DDIM loops and steps (b200mdm_set_joint_guidance), after set_cond,
        which clears it: mean / std [D], target [B, J, 3, T], weight [B, J, T], all on the engine's device."""
        ts = [t.to(torch.float32).contiguous() for t in (mean, std, target, weight)]
        check(self.lib.b200mdm_set_joint_guidance(self.h, *[_ptr(t) for t in ts], float(step), int(iters), _stream()))
        self._keep_guide(0, ts)

    def set_foot_guidance(self, contact_weight, floor_weight, floor_height=0.0, contact=None, lengths=None):
        """The foot-contact and floor terms of the joint guidance set last (b200mdm_set_foot_guidance), which
        set_joint_guidance and set_cond clear: contact [B, 4, T] on the engine's device or None (derived from each step's
        x0), lengths [B] or None (every frame)."""
        kappa = None if contact is None else contact.to(torch.float32).contiguous()
        n = _lengths_host(lengths, self.batch)
        check(self.lib.b200mdm_set_foot_guidance(self.h, float(contact_weight), float(floor_weight), float(floor_height),
                                                 None if kappa is None else _ptr(kappa),
                                                 None if n is None else n.ctypes.data_as(ctypes.c_void_p), _stream()))
        self._keep_guide(1, kappa)

    def set_scene_guidance(self, obstacle_weight, obstacle_margin, sdf=None, terrain=None):
        """The scene terms of the joint guidance set last (b200mdm_set_scene_guidance), after set_foot_guidance (whose
        lengths and floor they use), which set_joint_guidance, set_foot_guidance and set_cond clear: sdf / terrain
        SceneGrid or None, copied to the engine's device."""
        dev = torch.device("cuda", torch.cuda.current_device())
        (gs, vs), (gt, vt) = _grid(sdf, dev), _grid(terrain, dev)
        check(self.lib.b200mdm_set_scene_guidance(self.h, float(obstacle_weight), float(obstacle_margin), _grid_ref(gs),
                                                  _grid_ref(gt), _stream()))
        self._keep_guide(2, (vs, vt))

    def set_interaction_guidance(self, characters, weight, margin, placement, pairs=None, reach=None, pair_weight=None):
        """The interaction terms of the joint guidance set last (b200mdm_set_interaction_guidance), after
        set_scene_guidance or set_foot_guidance, whose terms and lengths they extend and which clear them, as do
        set_joint_guidance and set_cond: placement [B, 3], pairs int [N, 4] scene-local (a, j, b, k) or None, reach [N],
        pair_weight [N, T] or [B / C, N, T], copied to the engine's device."""
        dev = torch.device("cuda", torch.cuda.current_device())
        args, keep = _interaction(characters, weight, margin, placement, pairs, reach, pair_weight, dev)
        check(self.lib.b200mdm_set_interaction_guidance(self.h, *args, _stream()))
        self._keep_guide(3, keep)

    def set_cond_multi(self, batch, nframes, y, embed, action, weight, device):
        """Multi-prompt guidance (b200mdm_set_cond_multi / _dec / _tokens, then b200mdm_set_prompt_weight): embed fp32
        [K, B, C] (text models; for the BERT decoder a list of K (tokens [Mt_k, B, C], mask [B, Mt_k]) pairs) or action
        int64 numpy [B, K] (action models), weight fp32 [B, K, D or 1, T or 1], as MultiPromptSampleModel.prompts returns
        them; lengths and the target from y as set_cond takes them."""
        y = y or {}
        K = int(weight.shape[1])
        ln, _ = self._lengths_and_scale(batch, y, False, device)
        ln_p = None if ln is None else ln.ctypes.data_as(ctypes.c_void_p)
        n_tokens = 1
        if self.dec and not self.dec_clip:
            te, mask = self.prompt_memories(embed, batch, device)
            n_tokens = int(te.shape[1])
            check(self.lib.b200mdm_set_cond_multi_tokens(self.h, batch, nframes, K, _ptr(te),
                                                         mask.ctypes.data_as(ctypes.c_void_p), n_tokens, ln_p, _stream()))
            self._keep["cond_mask"] = mask
        else:
            te = None if embed is None else embed.detach().to(device=device, dtype=torch.float32).contiguous()
            if self.dec:
                check(self.lib.b200mdm_set_cond_multi_dec(self.h, batch, nframes, K, _ptr(te), ln_p, _stream()))
            else:
                ac = None if action is None else np.ascontiguousarray(action, dtype=np.int64)
                check(self.lib.b200mdm_set_cond_multi(self.h, batch, nframes, K, _ptr(te), ln_p,
                                                      None if ac is None else ac.ctypes.data_as(ctypes.c_void_p), _stream()))
        self._keep["cond"] = (te,)
        self.batch, self.nframes, self.halves, self.n_tokens, self.groups = batch, nframes, 1, n_tokens, K + 1
        self._set_target(batch, y, device)
        w = weight.detach().to(device=device, dtype=torch.float32).contiguous()
        strides = [0 if w.shape[i] == 1 else w.stride(i) for i in range(4)]
        check(self.lib.b200mdm_set_prompt_weight(self.h, K, _ptr(w), *strides, _stream()))
        self._keep["prompt_weight"] = w

    # ------------------------------------------------------------------ compute
    def denoise(self, x, timesteps):
        x = x.to(torch.float32).contiguous()
        ts = np.ascontiguousarray(timesteps.detach().reshape(-1).cpu().numpy().astype(np.int32))
        assert ts.shape[0] == x.shape[0]
        out = torch.empty_like(x)
        check(self.lib.b200mdm_denoise(self.h, _ptr(x), ts.ctypes.data_as(ctypes.c_void_p), _ptr(out), _stream()))
        return out

    def tap_shapes(self):
        """{tap name: (shape, dtype)} of every b200mdm_test_forward_taps point the current model and workspace have
        (include/b200mdm.h, B200MDM_TAP_*); each size is b200mdm_test_tap_bytes's, which is asserted."""
        c = self.cfg
        d, ff, L, B, T, Bp = c.latent_dim, c.ff_size, c.num_layers, self.batch, self.nframes, self.packed_batch()
        dip = self.dec and not self.dec_clip
        S = T + (self.context_len if dip else 1)
        M, kw, mem, h, f = Bp * S, 2 if dip else 1, Bp * self.n_tokens, torch.float16, torch.float32
        blend = Bp if self.groups else B           # multi-prompt guidance splits every group's frame rows as they are
        out = dict(EMBED=((M, 2 * d), h), TOK0=((M, 2 * d), h), TEMB=((B, d), f), L_IN=((M, 2 * d), h),
                   L_QKV=((M, 3 * d), h), L_ATT=((M, kw * d), h), L_LN1=((M, 2 * d), h), L_FFN=((M, kw * ff), h),
                   L_LN3=((M, 2 * d), h), BLEND=((blend * T, 3 * d), h))
        if not dip:
            out["CONDPROJ"] = ((Bp, d), f)
        if self.dec:
            out["L_LN2"] = ((M, 2 * d), h)
        if self.dec_clip:
            out["CROSS_C"] = ((L, Bp, d), f)
        if dip:
            out.update(MEM16=((mem, 2 * d), h), KVC16=((mem, L * 2 * d), h), L_QC=((M, d), h), L_XATT=((M, kw * d), h))
        if self.groups:
            out["X0G"] = ((Bp, c.njoints * c.nfeats, T), f)
        for i, name in enumerate(_lib.TAPS):
            n = int(self.lib.b200mdm_test_tap_bytes(self.h, i))
            if n < 0:
                check(n)
            want = int(np.prod(out[name][0])) * out[name][1].itemsize if name in out else 0
            assert n == want, "tap %s: the engine copies %d bytes, tap_shapes sizes %d" % (name, n, want)
        return out

    def forward_taps(self, x, timesteps, layer, names=None):
        """One forward as denoise() does, with the stage outputs of b200mdm_test_forward_taps: (out, {tap name: tensor})
        for the points in `names` (default: every point of this model), per-layer points at `layer`."""
        x = x.to(torch.float32).contiguous()
        ts = np.ascontiguousarray(timesteps.detach().reshape(-1).cpu().numpy().astype(np.int32))
        assert ts.shape[0] == x.shape[0]
        shapes = self.tap_shapes()
        taps = {n: torch.empty(*shapes[n][0], device=x.device, dtype=shapes[n][1]) for n in (names or shapes)}
        ptrs = (ctypes.c_void_p * len(_lib.TAPS))(*[taps[n].data_ptr() if n in taps else None for n in _lib.TAPS])
        out = torch.empty_like(x)
        check(self.lib.b200mdm_test_forward_taps(self.h, _ptr(x), ts.ctypes.data_as(ctypes.c_void_p), _ptr(out), int(layer),
                                                 ptrs, len(_lib.TAPS), _stream()))
        return out, taps

    def sample_step(self, mode, index, x_t, noise, flags=0, want_pred=True):
        """noise may be None for MODE_DDIM_REVERSE, which draws none."""
        x_t = x_t.to(torch.float32).contiguous()
        noise = noise.to(torch.float32).contiguous() if noise is not None else None
        out = torch.empty_like(x_t)
        pred = torch.empty_like(x_t) if want_pred else None
        check(self.lib.b200mdm_sample_step(self.h, mode, index, _ptr(x_t), _ptr(noise), flags, _ptr(out), _ptr(pred),
                                           _stream()))
        return out, pred

    def sample_step_at(self, mode, indices, x_t, noise, flags=0, want_pred=True):
        """One DDPM / DDIM step where sample b takes schedule index indices[b] (b200mdm_sample_step_at)."""
        idx = np.ascontiguousarray(np.asarray(indices).reshape(-1), dtype=np.int32)
        x_t = x_t.to(torch.float32).contiguous()
        noise = noise.to(torch.float32).contiguous()
        out = torch.empty_like(x_t)
        pred = torch.empty_like(x_t) if want_pred else None
        check(self.lib.b200mdm_sample_step_at(self.h, mode, idx.ctypes.data_as(ctypes.c_void_p), _ptr(x_t), _ptr(noise),
                                              flags, _ptr(out), _ptr(pred), _stream()))
        return out, pred

    # ------------------------------------------------------------------ continuous batching (serving.ContinuousSampler)
    def slots_begin(self, slots, nframes, guided, mode, flags=0):
        """A slot session on the (slots, nframes) workspace (b200mdm_slots_begin): every slot idle."""
        check(self.lib.b200mdm_slots_begin(self.h, int(slots), int(nframes), int(bool(guided)), mode, flags, _stream()))
        self.batch, self.nframes, self.halves, self.n_tokens = int(slots), int(nframes), 2 if guided else 1, 1
        self.groups = 0
        self._keep["slots"] = {}

    def slot_admit(self, slot, embed, action, scale, length, seed, sample_index):
        """One request into an idle slot (b200mdm_slot_admit): embed [cond_dim] fp32 on the device or None."""
        embed = embed.to(torch.float32).contiguous() if embed is not None else None
        check(self.lib.b200mdm_slot_admit(self.h, int(slot), _ptr(embed), int(action), float(scale), int(length),
                                          ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), int(sample_index), _stream()))
        self._keep["slots"][int(slot)] = embed      # read by the admission's kernels, which run asynchronously

    def slots_run(self, n_steps, use_graph=True):
        check(self.lib.b200mdm_slots_run(self.h, int(n_steps), int(use_graph), _stream()))

    def slot_read(self, slot, out):
        """out [njoints, nfeats, nframes] fp32 <- the finished sample of `slot`, which becomes free (b200mdm_slot_read)."""
        assert out.is_contiguous() and out.dtype == torch.float32
        check(self.lib.b200mdm_slot_read(self.h, int(slot), _ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ token-memory slots (serving.ContinuousChainSampler)
    def chain_slots_begin(self, slots, nframes, guided, mode, n_tokens, flags=0):
        """A slot session of a BERT-memory decoder with memories of n_tokens tokens (b200mdm_chain_slots_begin)."""
        check(self.lib.b200mdm_chain_slots_begin(self.h, int(slots), int(nframes), int(bool(guided)), mode, flags,
                                                 int(n_tokens), _stream()))
        self.batch, self.nframes, self.halves, self.n_tokens = int(slots), int(nframes), 2 if guided else 1, int(n_tokens)
        self.groups = 0
        self._keep["slots"] = {}

    def chain_slot_admit(self, slot, tokens, mask, prefix, scale, length, include_prefix, seed, sample_index):
        """One request into an idle slot (b200mdm_chain_slot_admit): tokens [n_tokens, cond_dim] fp32 and mask
        [n_tokens] uint8 (1 = padding) on the device, prefix [njoints * nfeats, context_len] fp32 on the device or None."""
        check(self.lib.b200mdm_chain_slot_admit(self.h, int(slot), _ptr(tokens), _ptr(mask), _ptr(prefix), float(scale),
                                                int(length), int(bool(include_prefix)),
                                                ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), int(sample_index), _stream()))
        self._keep["slots"][int(slot)] = (tokens, mask, prefix)   # read by kernels that run asynchronously

    def chain_slot_handoff(self, slot, out, tokens=None, mask=None):
        """The hand-off of a slot that has just finished a chunk (b200mdm_chain_slot_handoff): the chunk into out
        [njoints * nfeats, length], then the next chunk armed, with a new prompt when tokens / mask are given."""
        assert out.is_contiguous() and out.dtype == torch.float32
        check(self.lib.b200mdm_chain_slot_handoff(self.h, int(slot), _ptr(out), _ptr(tokens), _ptr(mask), _stream()))
        if tokens is not None:
            self._keep["slots"][int(slot)] = (tokens, mask)

    def sample_loop(self, mode, x, tape, skip_timesteps=0, flags=0, use_graph=True):
        """x: [B,J,F,T] fp32 (x_T, left untouched); tape: [n_run, B,J,F,T] fp32.  Returns x_0 (new tensor)."""
        x = x.to(torch.float32).contiguous()
        assert tape.is_contiguous() and tape.dtype == torch.float32
        out = torch.empty_like(x)
        check(self.lib.b200mdm_sample_loop(self.h, mode, skip_timesteps, _ptr(x), _ptr(out), _ptr(tape), tape.stride(0),
                                           flags, int(use_graph), _stream()))
        # the loop is asynchronous and runs on the engine's own stream, which torch's caching allocator knows nothing
        # about: the inputs are kept referenced here until the next loop replaces them
        self._keep["loop"] = (x, tape)
        return out

    def sample_loop_range(self, mode, first_index, n_run, x_in, x_out, tape, flags=0, use_graph=True):
        """Steps first_index .. first_index-n_run+1 on the engine's working buffer (b200mdm_sample_loop_range).
        x_in None: continue; x_out None: leave the state in the engine; tape None: B200MDM_FLAG_PHILOX_NOISE."""
        if tape is not None:
            assert tape.is_contiguous() and tape.dtype == torch.float32 and tape.shape[0] >= n_run
        else:
            flags |= _lib.FLAG_PHILOX_NOISE
        check(self.lib.b200mdm_sample_loop_range(self.h, mode, first_index, n_run, _ptr(x_in), _ptr(x_out), _ptr(tape),
                                                 tape.stride(0) if tape is not None else 0, flags, int(use_graph), _stream()))

    def ddim_reverse_loop_range(self, first_index, n_run, x_in, x_out, flags=0, use_graph=True):
        """DDIM inversion steps first_index .. first_index+n_run-1 on the engine's working buffer
        (b200mdm_ddim_reverse_loop_range).  x_in None: continue; x_out None: leave the state in the engine."""
        check(self.lib.b200mdm_ddim_reverse_loop_range(self.h, first_index, n_run, _ptr(x_in), _ptr(x_out), flags,
                                                       int(use_graph), _stream()))

    def plms_loop_range(self, order, first_index, n_run, x_in, x_out, flags=0, use_graph=True):
        """PLMS steps first_index .. first_index-n_run+1 on the engine's working buffer (b200mdm_plms_loop_range).
        x_in None: continue the previous PLMS loop; x_out None: leave the state in the engine."""
        check(self.lib.b200mdm_plms_loop_range(self.h, order, first_index, n_run, _ptr(x_in), _ptr(x_out), flags,
                                               int(use_graph), _stream()))

    def dpm_loop_range(self, order, first_index, n_run, x_in, x_out, flags=0, use_graph=True):
        """DPM-Solver++ steps first_index .. first_index-n_run+1 on the engine's working buffer (b200mdm_dpm_loop_range).
        x_in None: continue the previous DPM-Solver++ loop of this order; x_out None: leave the state in the engine."""
        check(self.lib.b200mdm_dpm_loop_range(self.h, order, first_index, n_run, _ptr(x_in), _ptr(x_out), flags,
                                              int(use_graph), _stream()))

    def vb_loop_range(self, first_index, n_run, x_start, tape, flags=0, terms=None, bpd=None, use_graph=True):
        """Bound steps first_index .. first_index-n_run+1 (b200mdm_vb_loop_range).  x_start None: continue the bound loop in
        the engine; tape None: B200MDM_FLAG_PHILOX_NOISE; terms [3, B, n_steps] / bpd [2, B] fp32 outputs or None."""
        if tape is not None:
            assert tape.is_contiguous() and tape.dtype == torch.float32 and tape.shape[0] >= n_run
        else:
            flags |= _lib.FLAG_PHILOX_NOISE
        check(self.lib.b200mdm_vb_loop_range(self.h, first_index, n_run, _ptr(x_start), _ptr(tape),
                                             tape.stride(0) if tape is not None else 0, flags, _ptr(terms), _ptr(bpd),
                                             int(use_graph), _stream()))

    def chain_setup(self, n_chunks, pred_len, include_prefix, crop, enc_chunks=None, mask_chunks=None):
        """An autoregressive chain of n_chunks prefix completions after set_cond (b200mdm_chain_setup): enc_chunks
        [n, Mt, B, C] fp32 device and mask_chunks uint8 numpy [n, B, Mt] give every chunk its memory (None: set_cond's)."""
        mask = None if mask_chunks is None else np.ascontiguousarray(mask_chunks, dtype=np.uint8)
        check(self.lib.b200mdm_chain_setup(self.h, int(n_chunks), int(pred_len), int(self.context_len), int(bool(include_prefix)),
                                           int(crop), _ptr(enc_chunks), None if mask is None else mask.ctypes.data_as(ctypes.c_void_p),
                                           _stream()))
        self._keep["chain"] = (enc_chunks, mask)

    def chain_set_goal(self, mean, std, goal, valid):
        """Goals in the world frame for the chain set up last (b200mdm_chain_set_goal): mean / std [D], goal
        [n_goals, B, n_ext, 3] (n_goals 1 or n_chunks) on the engine's device, valid uint8 numpy [B, n_ext]."""
        mean, std, goal = (t.to(torch.float32).contiguous() for t in (mean, std, goal))
        valid = np.ascontiguousarray(valid, dtype=np.uint8)
        check(self.lib.b200mdm_chain_set_goal(self.h, _ptr(mean), _ptr(std), _ptr(goal), int(goal.shape[0]),
                                              valid.ctypes.data_as(ctypes.c_void_p), _stream()))
        self._keep["goal"] = (mean, std, goal)

    @staticmethod
    def chunk_frame(carry, frames, mean, std, goal):
        """One chunk boundary of a goal-directed chain (b200mdm_chunk_frame): advances carry [B, 6] fp64 (in place) over
        frames [B, D, ..., n] (normalised; n may be 0) and returns goal [B, n_ext, 3] in the frame of the next frame."""
        lib = _lib.load()
        assert carry.dtype == torch.float64 and carry.is_contiguous()
        B, D, n = int(frames.shape[0]), int(frames.shape[1]), int(frames.shape[-1])
        frames = frames.to(torch.float32).reshape(B, D, n).contiguous()
        mean, std, goal = (t.to(torch.float32).contiguous() for t in (mean, std, goal))
        out = torch.empty_like(goal)
        check(lib.b200mdm_chunk_frame(_ptr(carry), _ptr(frames) if n > 0 else None, B, D, n, _ptr(mean), _ptr(std),
                                      _ptr(goal), int(goal.shape[1]), _ptr(out), _stream()))
        return out

    def chain_loop_range(self, mode, order, first_step, n_run, x_T, noise, out, flags=0, use_graph=True):
        """Global steps first_step .. first_step+n_run-1 of the chain (b200mdm_chain_loop_range).  x_T [n_chunks, ...]
        one per chunk, [...] one for every chunk, or None (the Philox x_T); noise [>= n_run, ...] or None (Philox eps, or
        none for DPM-Solver++).  out [B, J, F, crop] receives every chunk's frames."""
        if x_T is None or (noise is None and mode != _lib.MODE_DPM):
            flags |= _lib.FLAG_PHILOX_NOISE
        xs = 0 if x_T is None or x_T.dim() == out.dim() else x_T.stride(0)
        check(self.lib.b200mdm_chain_loop_range(self.h, mode, order, first_step, n_run, _ptr(x_T), xs, _ptr(noise),
                                                noise.stride(0) if noise is not None else 0, _ptr(out), flags,
                                                int(use_graph), _stream()))

    def dpm_pred_xstart(self, out):
        """out <- the x0 of the last step of the DPM-Solver++ loop in the engine (b200mdm_dpm_pred_xstart)."""
        check(self.lib.b200mdm_dpm_pred_xstart(self.h, _ptr(out), _stream()))
        return out

    def plms_step(self, index, order, x_t, old_eps, flags=0):
        """One plms_sample step (b200mdm_plms_step): old_eps = list of [B,J,F,T] eps, oldest first, possibly empty
        (an Adams-Bashforth step), or None (no old_out: the improved-Euler step).
        Returns (sample, pred_xstart, eps of this step)."""
        x_t = x_t.to(torch.float32).contiguous()
        old = [o.to(torch.float32).contiguous() for o in old_eps] if old_eps is not None else []
        ptrs = (ctypes.c_void_p * max(1, len(old)))(*[o.data_ptr() for o in old]) if old_eps is not None else None
        out, pred, eps = torch.empty_like(x_t), torch.empty_like(x_t), torch.empty_like(x_t)
        check(self.lib.b200mdm_plms_step(self.h, index, order, _ptr(x_t), ptrs, len(old), flags, _ptr(out), _ptr(pred),
                                         _ptr(eps), _stream()))
        self._keep["plms"] = (x_t, old)
        return out, pred, eps

    def set_noise_stream(self, seed, sample_index_base=0):
        check(self.lib.b200mdm_set_noise_stream(self.h, ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), int(sample_index_base)))

    def philox_normal(self, shape, seed, sample_index_base, step_id, device):
        """[B, ...] fp32 from the engine's counter-based stream (x_T: step_id = -1)."""
        out = torch.empty(tuple(shape), device=device, dtype=torch.float32)
        n = out[0].numel()
        check(self.lib.b200mdm_philox_normal(_ptr(out), int(shape[0]), n, ctypes.c_uint64(int(seed) & (2 ** 64 - 1)),
                                             int(sample_index_base), int(step_id), _stream()))
        return out

    def q_sample(self, sqrt_ac, sqrt_1mac, x_start, noise):
        out = torch.empty_like(noise)
        check(self.lib.b200mdm_q_sample(self.h, float(sqrt_ac), float(sqrt_1mac), _ptr(x_start), _ptr(noise), _ptr(out),
                                        noise.numel(), _stream()))
        return out

    def launch_count(self, reset=False):
        return int(self.lib.b200mdm_launch_count(self.h, int(reset)))
