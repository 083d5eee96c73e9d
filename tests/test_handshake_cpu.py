"""CPU: long motions from chained windows (HandshakeSampleModel, stitch_handshake, b200mdm_set_handshake).

  * the oracle's blend (oracle/handshake_oracle.py) against a direct numpy restatement: positions, weights, both
    copies, and motions that do not interact;
  * tests/golden/handshake_small.npz (the unmodified reference's samplers around the oracle's wrapper) against the fp32
    oracle run on the same inputs;
  * stitch_handshake's lengths and content; every validation error; the DiP, inversion and bound rejections; the
    shard-boundary check; the C ABI's argument checks, which run before any CUDA call."""
import ctypes
import importlib
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from b200mdm.utils.sampler_util import handshake_layout
from conftest import default_args, rel_err
from oracle import handshake_oracle as ho
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

gh = importlib.import_module("oracle.gen_golden_handshake")
deo = importlib.import_module("oracle.dec_emb_oracle")
LENGTHS, STARTS, H = [24, 20, 24, 16, 24], [1, 0, 0, 1, 0], 6


def test_oracle_blend_matches_numpy_restatement():
    g = torch.Generator().manual_seed(3)
    D = torch.randn(5, 7, 1, 24, generator=g, dtype=torch.float64)
    ms = torch.tensor(STARTS, dtype=torch.bool)
    out = ho.blend(D, H, torch.tensor(LENGTHS), ms)
    assert torch.allclose(out, torch.from_numpy(ho.blend_np(D.numpy(), H, LENGTHS, STARTS)), rtol=0, atol=1e-15)
    # positions and weights, written out: window 1 continues window 0 (n_0 = 24), window 4 continues window 3 (n_3 = 16)
    for p, b in ((0, 1), (1, 2), (3, 4)):
        n_p = LENGTHS[p]
        for j in range(H):
            a = (j + 1) / (H + 1)
            want = (1 - a) * D[p, ..., n_p - H + j] + a * D[b, ..., j]
            assert torch.allclose(out[p, ..., n_p - H + j], want, atol=1e-15)
            assert torch.equal(out[p, ..., n_p - H + j], out[b, ..., j])          # both copies
    # frames outside the handshakes are untouched; window 2 -> 3 is a motion boundary
    touched = torch.zeros(5, 24, dtype=torch.bool)
    for p, b in ((0, 1), (1, 2), (3, 4)):
        touched[p, LENGTHS[p] - H: LENGTHS[p]] = True
        touched[b, :H] = True
    assert torch.equal(out[..., ~touched[0]][0], D[0][..., ~touched[0]])
    assert not touched[2, LENGTHS[2] - H:].any() and not touched[3, :H].any()
    for b in range(5):
        assert torch.equal(out[b][..., ~touched[b]], D[b][..., ~touched[b]])
    # motions do not interact: changing motion 2 leaves motion 1 as it was
    D2 = D.clone()
    D2[3:] += 1.0
    assert torch.equal(ho.blend(D2, H, torch.tensor(LENGTHS), ms)[:3], out[:3])
    assert torch.equal(ho.blend(D, 0, torch.tensor(LENGTHS), ms), D)


def _small_oracle():
    c = gh.SMALL
    inp, shape, y = gh.small_inputs()
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    tmap = list(range(c["steps"]))
    return c, inp, shape, y, W, tabs, tmap


def test_fixtures_agree_with_the_oracle(golden):
    gold = golden("handshake_small.npz")
    c, inp, shape, y, W, tabs, tmap = _small_oracle()
    ln, ms, sc, te = y["lengths"], y["motion_start"], inp["scale"], inp["text_embed"]
    with torch.no_grad():
        guided = ho.denoiser(po.enc_denoiser(W, tmap, te, sc, ln), c["h"], ln, ms)
        bare = ho.denoiser(po.enc_denoiser(W, tmap, te, None, ln), c["h"], ln, ms)
        got = dict(fwd_guided=guided(inp["tape"][0], c["t_fwd"]), fwd_unguided=bare(inp["tape"][0], c["t_fwd"]),
                   ddpm=deo.sample_loop(guided, tabs, inp["tape"]),
                   ddim=deo.sample_loop(guided, tabs, inp["tape"], sampler="ddim"),
                   plms=po.plms_loop(guided, tabs, inp["tape"][0], order=2),
                   ddpm_inpaint=deo.sample_loop(guided, tabs, inp["tape"], inpaint=gh.inpaint_inputs(shape, c["inpaint_frames"])))
    for k, v in got.items():
        e = rel_err(v, gold[k])
        print("%s: oracle vs reference %.2e" % (k, e))
        assert e < 1e-5, (k, e)
    # the blend does something: the handshake frames differ from the plain model's
    plain = po.enc_denoiser(W, tmap, te, sc, ln)(inp["tape"][0], c["t_fwd"])
    assert rel_err(plain, gold["fwd_guided"]) > 1e-2


def test_stitch_lengths_and_content():
    B, T = 5, 24
    s = torch.arange(B * 2 * T, dtype=torch.float32).reshape(B, 2, 1, T)
    out = b200mdm.stitch_handshake(s, torch.tensor(LENGTHS), H, torch.tensor(STARTS, dtype=torch.bool))
    assert [tuple(m.shape) for m in out] == [(2, 1, 24 + 20 + 24 - 2 * H), (2, 1, 16 + 24 - H)]
    assert torch.equal(out[0], torch.cat([s[0, ..., :24], s[1, ..., H:20], s[2, ..., H:24]], -1))
    assert torch.equal(out[1], torch.cat([s[3, ..., :16], s[4, ..., H:24]], -1))
    one = b200mdm.stitch_handshake(s, None, H)
    assert len(one) == 1 and one[0].shape[-1] == B * T - (B - 1) * H
    assert [m.shape[-1] for m in b200mdm.stitch_handshake(s, None, 0, [1, 1, 1, 1, 1])] == [T] * B


@pytest.mark.parametrize("case", ["h_negative", "short_chained", "overlap", "first_not_start", "shape", "too_long"])
def test_validation_errors(case):
    B, T = 5, 24
    kw = dict(lengths=LENGTHS, motion_start=STARTS, h=H)
    if case == "h_negative":
        kw["h"] = -1
    elif case == "short_chained":
        kw["lengths"] = [24, 20, 24, 5, 24]            # window 3 is chained to window 4 and has 5 < 6 frames
    elif case == "overlap":
        kw["lengths"] = [24, 11, 24, 16, 24]           # window 1 has both neighbours and 11 < 12 frames
    elif case == "first_not_start":
        kw["motion_start"] = [0, 0, 0, 1, 0]
    elif case == "shape":
        kw["motion_start"] = [1, 0, 0, 1]
    else:
        kw["lengths"] = [24, 20, 25, 16, 24]
    with pytest.raises(ValueError):
        handshake_layout(B, T, kw["h"], kw["lengths"], kw["motion_start"])
    with pytest.raises(ValueError):
        b200mdm.stitch_handshake(torch.zeros(B, 2, 1, T), kw["lengths"], kw["h"], kw["motion_start"])
    # a window that begins a motion and has no successor in it may be short
    handshake_layout(B, T, H, [24, 20, 24, 3, 24], [1, 0, 0, 1, 1])
    handshake_layout(B, T, 0, [24, 1, 24, 3, 24], STARTS)


def _model(**over):
    return b200mdm.create_model_and_diffusion(default_args(layers=1, diffusion_steps=4, **over),
                                              SimpleNamespace(dataset=SimpleNamespace()))


def test_rejections():
    model, diffusion = _model()
    with pytest.raises(ValueError):
        b200mdm.HandshakeSampleModel(model, -1)
    with pytest.raises(TypeError):
        b200mdm.HandshakeSampleModel(SimpleNamespace(model=model), 4)
    dip, _ = _model(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    with pytest.raises(NotImplementedError):
        b200mdm.HandshakeSampleModel(dip, 4)
    hs = b200mdm.HandshakeSampleModel(b200mdm.ClassifierFreeSampleModel(model), 4)
    assert hs.njoints == 263 and hs.cond_mask_prob == 0.1 and hs.handshake_size == 4
    x = torch.zeros(2, 263, 1, 24)
    y = {"text_embed": torch.zeros(1, 2, 512)}
    t = torch.zeros(2, dtype=torch.long)
    for call in (lambda: diffusion.ddim_reverse_sample_loop(hs, x, model_kwargs={"y": y}),
                 lambda: diffusion.ddim_reverse_sample(hs, x, t, model_kwargs={"y": y}),
                 lambda: next(diffusion.ddim_reverse_sample_loop_progressive(hs, x, model_kwargs={"y": y})),
                 lambda: diffusion.calc_bpd_loop(hs, x, model_kwargs={"y": y})):
        with pytest.raises(NotImplementedError):
            call()


def test_shard_boundaries():
    y = {"motion_start": torch.tensor([1, 0, 0, 1, 0, 1], dtype=torch.bool), "lengths": torch.arange(6),
         "text_embed": torch.zeros(1, 6, 512)}
    a = parallel.shard_model_kwargs({"y": y}, 0, 3)["y"]
    b = parallel.shard_model_kwargs({"y": y}, 3, 6)["y"]
    assert a["motion_start"].tolist() == [True, False, False] and b["motion_start"].tolist() == [True, False, True]
    assert b["lengths"].tolist() == [3, 4, 5]
    for lo, hi in ((0, 2), (2, 6), (1, 3), (0, 4)):
        with pytest.raises(ValueError):
            parallel.shard_model_kwargs({"y": y}, lo, hi)
    parallel.shard_model_kwargs({"y": y}, 5, 6)


def test_c_abi_rejects_without_gpu():
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    ln = (ctypes.c_int64 * 5)(*LENGTHS)
    ms = (ctypes.c_uint8 * 5)(*STARTS)
    assert lib.b200mdm_set_handshake(None, H, ln, ms, None) == _lib.EINVAL

    def hook(h=H, lengths=ln, starts=ms, B=5, T=24, halves=2, scale=buf):
        return lib.b200mdm_test_blend_handshake(buf, scale, buf, B, T, 512, 1, halves, h, lengths, starts, None)
    assert hook(h=-1) == _lib.EINVAL and b"handshake size" in lib.b200mdm_last_error()
    assert hook(starts=(ctypes.c_uint8 * 5)(0, 0, 0, 1, 0)) == _lib.EINVAL and b"motion_start" in lib.b200mdm_last_error()
    assert hook(lengths=(ctypes.c_int64 * 5)(24, 20, 24, 5, 24)) == _lib.EINVAL and b"chained" in lib.b200mdm_last_error()
    assert hook(lengths=(ctypes.c_int64 * 5)(24, 11, 24, 16, 24)) == _lib.EINVAL and b"overlap" in lib.b200mdm_last_error()
    assert hook(lengths=(ctypes.c_int64 * 5)(24, 20, 25, 16, 24)) == _lib.EINVAL and b"outside" in lib.b200mdm_last_error()
    assert hook(scale=None) == _lib.EINVAL
    assert hook(B=0) == _lib.EINVAL
