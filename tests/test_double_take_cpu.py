"""CPU: refined transitions between chained windows (transition_layout, refine_transitions, soft inpainting).

  * the oracle (oracle/double_take_oracle.py) against an fp64 numpy restatement: the soft blend, the weights, the gather
    and the paste;
  * transition_layout's exact weights, source frames and paste ranges, against the oracle and written out, with h = 0
    and m = 1 among them; every layout error;
  * tests/golden/double_take_small.npz (the unmodified reference's samplers around the oracle's wrapper) against the
    fp32 oracle on the same inputs;
  * shard slicing of y['inpainting_weight']; the argument errors of the samplers and of refine_transitions, and the C
    ABI's, all raised before any CUDA call."""
import ctypes
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import default_args, rel_err
from oracle import double_take_oracle as dt
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

gd = importlib.import_module("oracle.gen_golden_double_take")
deo = importlib.import_module("oracle.dec_emb_oracle")
LENGTHS, STARTS = [24, 20, 24, 16, 24], [1, 0, 0, 1, 0]


def test_soft_blend_matches_numpy_restatement():
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(3, 7, 1, 10, generator=g) * 2
    motion = torch.randn(3, 7, 1, 10, generator=g)
    w = torch.rand(3, 7, 1, 10, generator=g)
    w[0, 0] = 0.0
    w[0, 1] = 1.0
    w[1, 0] = -0.5                                      # outside [0, 1]: the selects still apply
    w[1, 1] = 1.5
    got = dt.soft_inpaint(x0, w, motion)
    want = dt.soft_inpaint_np(x0.numpy(), w.numpy(), motion.numpy())
    assert np.allclose(got.double().numpy(), want, rtol=0, atol=4e-7 * (np.abs(x0.numpy()) + np.abs(motion.numpy())).max())
    assert torch.equal(got[0, 0], x0[0, 0]) and torch.equal(got[0, 1], motion[0, 1])
    assert torch.equal(got[1, 0], x0[1, 0]) and torch.equal(got[1, 1], motion[1, 1])
    clipped = dt.soft_inpaint(x0, w, motion, clip=True)
    assert torch.equal(clipped, got.clamp(-1, 1))
    # the mutants the kernel tests rely on differ from the expression
    assert not torch.equal(dt.soft_inpaint(x0, w, motion, swap=True), got)
    assert not torch.equal(dt.soft_inpaint(x0, w, motion, clamp_first=True, clip=True), clipped)


@pytest.mark.parametrize("h,m", [(4, 3), (0, 1), (0, 5), (6, 1), (20, 10)])
def test_weights_exact(h, m):
    Lt = 2 * m + h
    w = b200mdm.transition_layout(2, 200, h, m)["weight"]
    assert w.dtype == np.float32 and w.shape == (Lt,)
    want = np.array([(m - f) / m if f < m else 0.0 if f < m + h else (f - m - h + 1) / m for f in range(Lt)])
    assert np.array_equal(w, want.astype(np.float32))
    assert torch.equal(torch.from_numpy(w), dt.weights(h, m))
    assert w[0] == 1.0 and w[-1] == 1.0 and (w[m:m + h] == 0).all()
    if m == 1:
        assert np.array_equal(w, np.array([1.0] + [0.0] * h + [1.0], dtype=np.float32))


@pytest.mark.parametrize("h,m", [(4, 3), (0, 1), (6, 2)])
def test_gather_and_paste(h, m):
    B, T = 5, 24
    ln, ms = torch.tensor(LENGTHS), torch.tensor(STARTS, dtype=torch.bool)
    lay = b200mdm.transition_layout(B, T, h, m, ln, ms)
    Lt = 2 * m + h
    assert lay["pairs"].tolist() == [[0, 1], [1, 2], [3, 4]]
    assert lay["motion"].tolist() == [0, 0, 1]
    # s = where b's handshake begins in its motion: 24 - h for window 1, 24 + 20 - 2h for window 2, 16 - h for window 4
    s = [24 - h, 24 + 20 - 2 * h, 16 - h]
    assert lay["paste"].tolist() == [[v - m + 1, v + h + m - 1] for v in s]
    for i, (p, b) in enumerate(lay["pairs"]):
        n_p = LENGTHS[p]
        assert lay["src_window"][i].tolist() == [p] * (m + h) + [b] * m
        assert lay["src_frame"][i].tolist() == [n_p - h - m + f for f in range(m + h)] + list(range(h, h + m))
    W = torch.arange(B * 2 * T, dtype=torch.float32).reshape(B, 2, 1, T)
    sw, sf = torch.from_numpy(lay["src_window"]), torch.from_numpy(lay["src_frame"])
    x_init = W[sw, :, :, sf].permute(0, 2, 3, 1)
    assert torch.equal(x_init, dt.gather(W, ln, ms, h, m))
    # every gathered frame is the stitched motion's frame s - m + f: the transition is a piece of the first take
    motions = b200mdm.stitch_handshake(W, ln, h, ms)
    for i, v in enumerate(s):
        assert torch.equal(x_init[i], motions[lay["motion"][i]][..., v - m: v - m + Lt])
    refined = -1 - torch.arange(3 * 2 * Lt, dtype=torch.float32).reshape(3, 2, 1, Lt)
    want = dt.paste(dt.stitch(W, ln, ms, h), refined, ln, ms, h, m)
    for i, (a, b) in enumerate(lay["paste"]):
        motions[lay["motion"][i]][..., a:b] = refined[i, ..., 1:Lt - 1]
    assert all(torch.equal(x, y) for x, y in zip(motions, want))


@pytest.mark.parametrize("case", ["m_zero", "short_one_side", "short_both_sides", "too_long", "h_negative"])
def test_layout_errors(case):
    B, T, h, m, ln = 5, 24, 4, 3, list(LENGTHS)
    kw = {}
    if case == "m_zero":
        m = 0
    elif case == "short_one_side":
        ln = [24, 20, 24, 6, 24]                          # window 3 is chained to window 4 and has 6 < h + m = 7
    elif case == "short_both_sides":
        ln = [24, 13, 24, 16, 24]                         # window 1 has both neighbours and 13 < 2h + 2m = 14
    elif case == "too_long":
        kw["max_frames"] = 2 * m + h - 1
    else:
        h = -1
    with pytest.raises(ValueError):
        b200mdm.transition_layout(B, T, h, m, ln, STARTS, **kw)
    # at the limits, and a short window that is chained on no side
    b200mdm.transition_layout(B, T, 4, 3, [24, 14, 24, 7, 24], STARTS)
    b200mdm.transition_layout(B, T, 4, 3, [24, 20, 24, 2, 24], [1, 0, 0, 1, 1])
    b200mdm.transition_layout(B, T, 4, 3, LENGTHS, STARTS, max_frames=10)
    assert b200mdm.transition_layout(B, T, 4, 3, LENGTHS, [1] * 5)["pairs"].shape == (0, 2)


def _oracle_take2(W, tabs, tmap, te, sc, ln, x_init, tape, c, sampler, clip=False, dec=False):
    """The reference's loop restated on the fp32 oracle: q_sample of x_init, then steps n - 1 - k .. 0."""
    w = dt.weights(c["h"], c["m"]).view(1, 1, 1, -1).expand_as(x_init)
    if dec:
        base = deo.denoiser(W, tmap, te, sc, ln)
    else:
        base = po.enc_denoiser(W, tmap, te, sc, ln)
    den = dt.denoiser(base, w, x_init)
    idx = list(range(c["steps"] - c["k"]))[::-1]
    if sampler == "plms":
        return po.plms_loop(den, tabs, tape[0], order=2, skip_timesteps=c["k"], init_image=x_init)
    x = mo.q_sample(tabs, x_init, idx[0], tape[0])
    for j, i in enumerate(idx):
        x0 = po.p_mean_x0(den(x, i), clip)
        x = mo.p_sample_step(tabs, x0, x, i, tape[1 + j])[0] if sampler == "ddpm" else mo.ddim_step(tabs, x0, x, i, tape[1 + j])
    return x


def test_fixture_agrees_with_the_oracle(golden):
    gold = golden("double_take_small.npz")
    c = gd.SMALL
    inp, y = gd.window_inputs()
    ln, ms = y["lengths"], y["motion_start"]
    x_init = dt.gather(gd.windows(), ln, ms, c["h"], c["m"])
    assert np.array_equal(x_init.numpy(), gold["x_init"])
    tape = gd.take2_tape(x_init.shape[0])
    yt = dt.transition_y(y, ln, ms, c["h"], c["m"], x_init)
    assert yt["scale"].tolist() == [1.0, 7.5, 4.0]
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    tmap = list(range(c["steps"]))
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    Wd = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=512,
                                                       seed=c["dec_weights_seed"]), c["L"], arch="trans_dec")
    args = (tabs, tmap, yt["text_embed"], yt["scale"], yt["lengths"])
    with torch.no_grad():
        got = dict(enc_ddpm=_oracle_take2(W, *args, x_init, tape, c, "ddpm"),
                   enc_ddim=_oracle_take2(W, *args, x_init, tape, c, "ddim"),
                   enc_plms=_oracle_take2(W, *args, x_init, tape, c, "plms"),
                   enc_ddpm_clip=_oracle_take2(W, *args, x_init, tape, c, "ddpm", clip=True),
                   dec_ddpm=_oracle_take2(Wd, *args, x_init, tape, c, "ddpm", dec=True))
    for k, v in got.items():
        e = rel_err(v, gold[k])
        print("%s: oracle vs reference %.2e" % (k, e))
        assert e < 1e-5, (k, e)
    # the anchors are pinned: DDPM's last step returns x0, which is the first take where w = 1
    for k in ("enc_ddpm", "dec_ddpm"):
        assert np.array_equal(gold[k][..., 0], gold["x_init"][..., 0]) and np.array_equal(gold[k][..., -1], gold["x_init"][..., -1])
    # the end-to-end motions are take 1 stitched, with take 2's inner frames pasted
    t1, t2 = torch.from_numpy(gold["e2e_take1"]), torch.from_numpy(gold["e2e_take2"])
    want = dt.paste(dt.stitch(t1, ln, ms, c["h"]), t2, ln, ms, c["h"], c["m"])
    assert all(np.array_equal(gold["e2e_motion%d" % i], w.numpy()) for i, w in enumerate(want))


def test_shard_slicing():
    w = torch.rand(6, 263, 1, 10)
    y = {"inpainting_weight": w, "inpainted_motion": torch.rand(6, 263, 1, 10), "text_embed": torch.zeros(1, 6, 512)}
    part = parallel.shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(part["inpainting_weight"], w[2:5]) and part["inpainted_motion"].shape[0] == 3


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


@pytest.mark.parametrize("case", ["both", "no_motion", "shape", "nan", "above", "below", "int"])
def test_sampler_argument_errors_before_the_engine(case):
    """The model stays on the CPU: any engine call would raise RuntimeError, so a ValueError comes first."""
    model, diffusion = _model()
    shape = (2, 263, 1, 10)
    w, motion = torch.full(shape, 0.5), torch.zeros(shape)
    y = {"text_embed": torch.zeros(1, 2, 512), "inpainting_weight": w, "inpainted_motion": motion}
    if case == "both":
        y["inpainting_mask"] = torch.zeros(shape, dtype=torch.bool)
    elif case == "no_motion":
        del y["inpainted_motion"]
    elif case == "shape":
        y["inpainting_weight"] = torch.full((2, 263, 1, 9), 0.5)
    elif case == "nan":
        w[0, 0, 0, 3] = float("nan")
    elif case == "above":
        w[1, 5, 0, 0] = 1.0001
    elif case == "below":
        w[1, 5, 0, 0] = -1e-30
    else:
        y["inpainting_weight"] = torch.ones(shape, dtype=torch.int32)
    x = torch.zeros(shape)
    t = torch.zeros(2, dtype=torch.long)
    kw = {"y": y}
    for call in (lambda: diffusion.p_sample_loop(model, shape, model_kwargs=kw),
                 lambda: diffusion.ddim_sample_loop(model, shape, model_kwargs=kw),
                 lambda: diffusion.plms_sample_loop(model, shape, model_kwargs=kw),
                 lambda: diffusion.dpm_solver_sample_loop(model, shape, model_kwargs=kw),
                 lambda: diffusion.p_sample(model, x, t, model_kwargs=kw),
                 lambda: next(diffusion.p_sample_loop_progressive(model, shape, noise=x, model_kwargs=kw)),
                 lambda: diffusion.ddim_reverse_sample_loop(model, x, model_kwargs=kw),
                 lambda: diffusion.p_mean_variance(model, x, t, model_kwargs=kw),
                 lambda: diffusion.calc_bpd_loop(model, x, model_kwargs=kw)):
        with pytest.raises(ValueError):
            call()


def test_refine_transitions_rejections():
    model, diffusion = _model()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    windows = torch.zeros(5, 263, 1, 24)
    y = {"text_embed": torch.zeros(1, 5, 512), "lengths": torch.tensor(LENGTHS),
         "motion_start": torch.tensor(STARTS, dtype=torch.bool), "scale": torch.ones(5)}
    kw = {"y": y}
    with pytest.raises(TypeError):
        b200mdm.refine_transitions(diffusion.ddim_sample_loop, b200mdm.HandshakeSampleModel(cfg, 4), windows, kw, 4, 3, 2)
    dip, _ = _model(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    with pytest.raises(NotImplementedError):
        b200mdm.refine_transitions(diffusion.ddim_sample_loop, dip, windows, kw, 4, 3, 2)
    for k in (-1, 4):
        with pytest.raises(ValueError):
            b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, windows, kw, 4, 3, k)
    with pytest.raises(ValueError):
        b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, windows, kw, 4, 0, 2)
    with pytest.raises(ValueError):
        b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, windows, kw, 4, 200, 2)
    # no chained pair: stitch_handshake's motions, no engine call (the model is on the CPU)
    singles = dict(y, motion_start=torch.ones(5, dtype=torch.bool))
    got = b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, windows + 1, {"y": singles}, 4, 3, 2)
    assert [m.shape[-1] for m in got] == LENGTHS and all(bool((m == 1).all()) for m in got)


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    handle = ctypes.c_void_p(ctypes.addressof(buf))    # never dereferenced: the pointer check comes first
    assert lib.b200mdm_set_inpaint_weight(None, buf, buf) == _lib.EINVAL
    assert lib.b200mdm_set_inpaint_weight(handle, buf, None) == _lib.EINVAL and b"both" in lib.b200mdm_last_error()
    assert lib.b200mdm_set_inpaint_weight(handle, None, buf) == _lib.EINVAL

    def hook(mode=_lib.MODE_DDPM, flags=0, weight=buf, motion=buf, B=2, halves=2, scale=buf):
        return lib.b200mdm_test_out_weight(buf, scale, buf, buf, buf, mode, flags, weight, motion, buf, B, 263, 10, 512, 1,
                                           halves, None)
    for mode in (4, 5, 9, -1):                        # PLMS improved Euler is not a family of its own; unknown modes
        assert hook(mode=mode) == _lib.EINVAL
    assert hook(weight=None) == _lib.EINVAL and hook(motion=None) == _lib.EINVAL
    assert hook(flags=_lib.FLAG_CONST_NOISE) == _lib.EINVAL
    assert hook(scale=None) == _lib.EINVAL and hook(B=0) == _lib.EINVAL
