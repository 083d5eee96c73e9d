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
        self._next_key = None
        self.batch = self.nframes = self.n_tokens = 0
        self.halves = 1

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
        self._next_key = None                     # the engine marks the reverse, DPM-Solver++ and bound tables stale
        self._dpm_key = None
        self._vb_key = None

    def set_schedule_next(self, rows, key=None):
        """[n_steps, 2] fp32 rows sqrt(abn), sqrt(1 - abn) of the current schedule (b200mdm_set_schedule_next)."""
        if key is not None and key == self._next_key:
            return
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        assert rows.ndim == 2 and rows.shape[1] == _lib.SCHED_NEXT_STRIDE
        check(self.lib.b200mdm_set_schedule_next(self.h, rows.shape[0], rows.ctypes.data_as(ctypes.c_void_p)))
        self._next_key = key

    def set_schedule_dpm(self, rows, key=None):
        """[n_steps, 4] fp32 rows c_x, c0, c_cur, c_prev of the current schedule (b200mdm_set_schedule_dpm)."""
        if key is not None and key == self._dpm_key:
            return
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        assert rows.ndim == 2 and rows.shape[1] == _lib.SCHED_DPM_STRIDE
        check(self.lib.b200mdm_set_schedule_dpm(self.h, rows.shape[0], rows.ctypes.data_as(ctypes.c_void_p)))
        self._dpm_key = key

    def set_schedule_vb(self, rows, key=None):
        """[n_steps, 12] fp32 rows of the variational-bound table of the current schedule (b200mdm_set_schedule_vb)."""
        if key is not None and key == getattr(self, "_vb_key", None):
            return
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        assert rows.ndim == 2 and rows.shape[1] == _lib.SCHED_VB_STRIDE
        check(self.lib.b200mdm_set_schedule_vb(self.h, rows.shape[0], rows.ctypes.data_as(ctypes.c_void_p)))
        self._vb_key = key

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

    def test_cross_rows(self, timestep, halves, device):
        """The CLIP decoder's per-step cross-attention rows (b200mdm_test_cross_rows) for the conditioning last set:
        [num_layers, halves * batch, d] fp32 at model timestep `timestep`."""
        out = torch.empty(self.cfg.num_layers, halves * self.batch, self.cfg.latent_dim, device=device, dtype=torch.float32)
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

    def _set_cond_dec(self, batch, nframes, y, guided, device):
        """DiP: y['text_embed'] = (BERT tokens [Mt,B,768], padding mask [B,Mt] True = pad), y['prefix'] [B,J,F,ctx]
        (reference model/mdm.py:203-206,210-217,264)."""
        if self.dec_clip:
            return self._set_cond_dec_clip(batch, nframes, y, guided, device)
        te = y.get("text_embed")
        if not isinstance(te, tuple):
            raise RuntimeError("trans_dec (DiP) needs y['text_embed'] = (tokens, mask) from bert_encode_text "
                               "(model/mdm.py:180-187)")
        enc, tmask = te
        enc = enc.detach().to(device=device, dtype=torch.float32)
        if enc.shape[1] == 1 and batch > 1:
            enc = enc.expand(-1, batch, -1)
        enc = enc.contiguous()
        if tmask.shape[0] == 1 and batch > 1:                  # model/mdm.py:215-216
            tmask = torch.repeat_interleave(tmask, batch, dim=0)
        Mt = enc.shape[0]
        assert enc.shape == (Mt, batch, self.cfg.cond_dim) and tuple(tmask.shape) == (batch, Mt), (enc.shape, tmask.shape)
        tm = np.ascontiguousarray(tmask.detach().cpu().numpy().astype(np.uint8))
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

    def set_inpaint(self, mask, motion):
        if mask is None:
            check(self.lib.b200mdm_set_inpaint(self.h, None, None))
            self._keep.pop("inpaint", None)
            return
        m8 = mask.to(torch.uint8).contiguous()
        mo = motion.to(torch.float32).contiguous()
        check(self.lib.b200mdm_set_inpaint(self.h, _ptr(m8), _ptr(mo)))
        self._keep["inpaint"] = (m8, mo)

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
        (include/b200mdm.h, B200MDM_TAP_*)."""
        c = self.cfg
        d, ff, L, B, T, Bp = c.latent_dim, c.ff_size, c.num_layers, self.batch, self.nframes, self.halves * self.batch
        dip = self.dec and not self.dec_clip
        S = T + (self.context_len if dip else 1)
        M, kw, mem, h, f = Bp * S, 2 if dip else 1, Bp * self.n_tokens, torch.float16, torch.float32
        out = dict(EMBED=((M, 2 * d), h), TOK0=((M, 2 * d), h), TEMB=((B, d), f), L_IN=((M, 2 * d), h),
                   L_QKV=((M, 3 * d), h), L_ATT=((M, kw * d), h), L_LN1=((M, 2 * d), h), L_FFN=((M, kw * ff), h),
                   L_LN3=((M, 2 * d), h), BLEND=((B * T, 3 * d), h))
        if not dip:
            out["CONDPROJ"] = ((Bp, d), f)
        if self.dec:
            out["L_LN2"] = ((M, 2 * d), h)
        if self.dec_clip:
            out["CROSS_C"] = ((L, Bp, d), f)
        if dip:
            out.update(MEM16=((mem, 2 * d), h), KVC16=((mem, L * 2 * d), h), L_QC=((M, d), h), L_XATT=((M, kw * d), h))
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
