"""GPU: refined transitions between chained windows (refine_transitions) and soft inpainting in the output epilogue.

  * the weighted x0 of every update family's epilogue (b200mdm_test_out_weight) bit for bit against an fp32 torch
    restatement, with the clamp on and off and weights that include exact 0 and 1; four mutants of the restatement (w and
    1 - w swapped, the clamp before the blend, the neighbouring sample's motion, a weight indexed by (b, t) only) differ;
  * 0 / 1 weights give the bool mask's loop and all-zero weights the loop without inpainting, bit for bit, for DDPM,
    DDIM, PLMS, DPM-Solver++, DDIM inversion and the variational bound, with the step graph and eagerly;
  * every entry of tests/golden/double_take_small.npz (the unmodified reference's samplers around the oracle's wrapper)
    within 1e-3 relative, refine_transitions end to end on the reference's take 1 among them; DPM-Solver++ against
    oracle/dpm_oracle.py around the wrapper, with h = 0 and m = 1 among the layouts;
  * engine state: soft -> bool -> none -> soft on one engine equals fresh engines; b200mdm_set_cond clears the weight;
    b200mdm_denoise ignores it."""
import ctypes
import importlib
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib
from conftest import default_args, rel_err
from oracle import double_take_oracle as dt
from oracle import dpm_oracle as do
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
gd = importlib.import_module("oracle.gen_golden_double_take")
FAMILIES = [_lib.MODE_X0, _lib.MODE_DDPM, _lib.MODE_DDIM, _lib.MODE_PLMS_AB, _lib.MODE_DDIM_REVERSE, _lib.MODE_DPM,
            _lib.MODE_VB]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _model(layers, steps, seed, guided=True, **over):
    args = default_args(layers=layers, diffusion_steps=steps, **over)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    kw = dict(arch="trans_dec", cond_dim=512) if over.get("arch") == "trans_dec" else {}
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=layers, seed=seed, **kw))
    model.to("cuda").eval()
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), diffusion


# ------------------------------------------------------------------------------------------------ the epilogue alone
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("mode", FAMILIES)
def test_weighted_epilogue_bit_exact(mode, clip):
    lib = _lib.load()
    B, JF, T, d, s_off, halves = 3, 263, 40, 512, 1, 2
    S = T + s_off
    g = torch.Generator(device="cuda").manual_seed(31 + mode)
    h = torch.randn(halves * B * S, d, device="cuda", generator=g) * 1.2
    hh = h.half()
    hres = torch.cat([hh, (h - hh.float()).half()], 1).contiguous()
    scale = torch.tensor([2.5, 7.5, 1.0], device="cuda")
    w_out = torch.randn(JF, d, device="cuda", generator=g) / d ** 0.5
    b_out = torch.randn(JF, device="cuda", generator=g) * 0.1
    xt = torch.randn(B, JF, T, device="cuda", generator=g)
    motion = torch.rand(B, JF, T, device="cuda", generator=g) * 2.4 - 1.2
    w = torch.rand(B, JF, T, device="cuda", generator=g)
    w[:, :, :6] = 0.0
    w[:, :, 6:12] = 1.0
    w[:, 5] = 0.0
    w[:, 7] = 1.0

    def x0(weight, flags):
        out = torch.full_like(xt, float("nan"))
        _lib.check(lib.b200mdm_test_out_weight(_p(hres), _p(scale), _p(w_out), _p(b_out), _p(xt), mode, flags, _p(weight),
                                               _p(motion if weight is not None else None), _p(out), B, JF, T, d, s_off,
                                               halves, _stream()))
        torch.cuda.synchronize()
        return out
    raw = x0(None, 0)                                                 # acc + bias, the operand of the blend
    got = x0(w, _lib.FLAG_CLIP_DENOISED if clip else 0)
    want = dt.soft_inpaint(raw, w, motion, clip=clip)
    assert torch.equal(got, want), float((got - want).abs().max())
    kept = motion.clamp(-1, 1) if clip else motion
    assert torch.equal(got[w >= 1], kept[w >= 1])
    mutants = dict(swap=dt.soft_inpaint(raw, w, motion, swap=True, clip=clip),
                   neighbour=dt.soft_inpaint(raw, w, motion.roll(1, 0), clip=clip),
                   bt_only=dt.soft_inpaint(raw, w[:, :1].expand_as(w), motion, clip=clip))
    if clip:
        mutants["clamp_first"] = dt.soft_inpaint(raw, w, motion, clamp_first=True, clip=True)
    for k, v in mutants.items():
        assert not torch.equal(got, v), k


# ------------------------------------------------------------------------------------------------ against the bool mask
@pytest.fixture(scope="module")
def small():
    L, steps, B, T = 2, 6, 3, 20
    cfg, diffusion = _model(L, steps, 3)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=41, lengths=[20, 14, 20], scale=torch.tensor([2.5, 7.5, 1.0]))
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    shape = (B, 263, 1, T)
    g = torch.Generator(device="cuda").manual_seed(9)
    mask = torch.rand(shape, device="cuda", generator=g) < 0.4
    motion = torch.rand(shape, device="cuda", generator=g) * 2 - 1
    return cfg, diffusion, inp, y, shape, mask, motion


def _run(diffusion, m, sampler, shape, y, xT, tape, use_graph):
    kw = dict(clip_denoised=True, model_kwargs={"y": y})
    if sampler == "ddpm":
        return diffusion.p_sample_loop(m, shape, noise=xT, noise_tape=tape, use_graph=use_graph, **kw)
    if sampler == "ddim":
        return diffusion.ddim_sample_loop(m, shape, noise=xT, noise_tape=tape, use_graph=use_graph, **kw)
    if sampler == "plms":
        return diffusion.plms_sample_loop(m, shape, noise=xT, use_graph=use_graph, **kw)
    if sampler == "dpm":
        return diffusion.dpm_solver_sample_loop(m, shape, noise=xT, use_graph=use_graph, **kw)
    if sampler == "reverse":
        return diffusion.ddim_reverse_sample_loop(m, xT, use_graph=use_graph, **kw)
    out = diffusion.calc_bpd_loop(m, xT, noise_tape=tape, use_graph=use_graph, **kw)
    return torch.cat([out["vb"], out["xstart_mse"], out["mse"]])


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("sampler", ["ddpm", "ddim", "plms", "dpm", "reverse", "vb"])
def test_binary_weights_are_the_bool_mask(small, sampler, use_graph):
    cfg, diffusion, inp, y, shape, mask, motion = small
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    with_mask = _run(diffusion, cfg, sampler, shape, dict(y, inpainting_mask=mask, inpainted_motion=motion), xT, tape, use_graph)
    soft = _run(diffusion, cfg, sampler, shape, dict(y, inpainting_weight=mask.float(), inpainted_motion=motion), xT, tape,
                use_graph)
    plain = _run(diffusion, cfg, sampler, shape, y, xT, tape, use_graph)
    zero = _run(diffusion, cfg, sampler, shape, dict(y, inpainting_weight=torch.zeros(shape, device="cuda"),
                                                     inpainted_motion=motion), xT, tape, use_graph)
    torch.cuda.synchronize()
    assert torch.equal(soft, with_mask) and torch.equal(zero, plain)
    assert not torch.equal(soft, plain)


def test_single_steps_and_progressive(small):
    cfg, diffusion, inp, y, shape, mask, motion = small
    x = inp["tape"][1].cuda()
    t = torch.full((shape[0],), 2, dtype=torch.long, device="cuda")
    ym, yw = dict(y, inpainting_mask=mask, inpainted_motion=motion), dict(y, inpainting_weight=mask.float(), inpainted_motion=motion)
    for fn in (lambda yy: diffusion.p_sample(cfg, x, t, model_kwargs={"y": yy}, noise=x)["pred_xstart"],
               lambda yy: diffusion.ddim_sample(cfg, x, t, model_kwargs={"y": yy}, noise=x)["sample"],
               lambda yy: diffusion.plms_sample(cfg, x, t, model_kwargs={"y": yy})["sample"],
               lambda yy: diffusion.p_mean_variance(cfg, x, t, model_kwargs={"y": yy})["mean"],
               lambda yy: list(diffusion.dpm_solver_sample_loop_progressive(cfg, shape, noise=x, model_kwargs={"y": yy}))[-1]["pred_xstart"]):
        assert torch.equal(fn(ym), fn(yw))


# ------------------------------------------------------------------------------------------------ parity
@pytest.fixture(scope="module")
def fixture_case():
    c = gd.SMALL
    inp, y = gd.window_inputs()
    ln, ms = y["lengths"], y["motion_start"]
    x_init = dt.gather(gd.windows(), ln, ms, c["h"], c["m"])
    tape = gd.take2_tape(x_init.shape[0])
    return c, inp, y, x_init, tape


def _cuda_y(y):
    return {k: v.cuda() if torch.is_tensor(v) else v for k, v in y.items()}


def test_fixture_parity(golden, fixture_case):
    gold = golden("double_take_small.npz")
    c, inp, y, x_init, tape = fixture_case
    ln, ms = y["lengths"], y["motion_start"]
    cfg, diffusion = _model(c["L"], c["steps"], c["weights_seed"])
    dec, ddiff = _model(c["L"], c["steps"], c["dec_weights_seed"], arch="trans_dec", emb_trans_dec=True, text_encoder_type="clip")
    yt = _cuda_y(dt.transition_y(y, ln, ms, c["h"], c["m"], x_init))
    xi, xT, eps = x_init.cuda(), tape[0].cuda(), torch.stack(tape[1:]).cuda()
    shape = tuple(x_init.shape)
    kw = dict(skip_timesteps=c["k"], init_image=xi, noise=xT, clip_denoised=False, model_kwargs={"y": yt})
    got = dict(enc_ddpm=diffusion.p_sample_loop(cfg, shape, noise_tape=eps, **kw),
               enc_ddim=diffusion.ddim_sample_loop(cfg, shape, eta=0.0, noise_tape=eps, **kw),
               enc_plms=diffusion.plms_sample_loop(cfg, shape, order=2, **kw),
               enc_ddpm_clip=diffusion.p_sample_loop(cfg, shape, noise_tape=eps, **dict(kw, clip_denoised=True)),
               dec_ddpm=ddiff.p_sample_loop(dec, shape, noise_tape=eps, **kw))
    # end to end: the engine's take 1 of the windows, then refine_transitions on the reference's take 1
    xw, tw = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    yw = _cuda_y(y)
    got["e2e_take1"] = diffusion.p_sample_loop(b200mdm.HandshakeSampleModel(cfg, c["h"]), (c["B"], 263, 1, c["T"]), noise=xw,
                                               clip_denoised=False, model_kwargs={"y": yw}, noise_tape=tw)
    motions = b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, torch.from_numpy(gold["e2e_take1"]).cuda(),
                                         {"y": yw}, c["h"], c["m"], c["k"], noise=xT, noise_tape=eps, clip_denoised=False,
                                         eta=0.0)
    for i, mo_ in enumerate(motions):
        got["e2e_motion%d" % i] = mo_
    for k, v in got.items():
        e = rel_err(v, gold[k])
        print("%s: engine vs reference %.2e" % (k, e))
        assert e < RTOL, (k, e)


@pytest.mark.parametrize("h,m", [(4, 3), (0, 1), (0, 3), (6, 1)])
@pytest.mark.parametrize("order", [1, 2])
def test_refine_transitions_dpm_vs_oracle(fixture_case, h, m, order):
    c, inp, y, _, _ = fixture_case
    ln, ms = y["lengths"], y["motion_start"]
    cfg, diffusion = _model(c["L"], c["steps"], c["weights_seed"])
    W = gd.windows()
    x_init = dt.gather(W, ln, ms, h, m)
    xT = torch.randn(x_init.shape, generator=torch.Generator().manual_seed(5 + h + m))
    motions = b200mdm.refine_transitions(diffusion.dpm_solver_sample_loop, cfg, W.cuda(), {"y": _cuda_y(y)}, h, m, c["k"],
                                         noise=xT.cuda(), clip_denoised=False, order=order)
    Wo = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    yt = dt.transition_y(y, ln, ms, h, m, x_init)
    w = yt["inpainting_weight"]
    den = dt.denoiser(po.enc_denoiser(Wo, list(range(c["steps"])), yt["text_embed"], yt["scale"], yt["lengths"]), w, x_init)
    with torch.no_grad():
        ref = do.dpm_loop(den, tabs, xT, order=order, skip_timesteps=c["k"], init_image=x_init)
    want = dt.paste(dt.stitch(W, ln, ms, h), ref, ln, ms, h, m)
    for got, wm in zip(motions, want):
        e = rel_err(got, wm)
        print("h %d m %d order %d: engine vs oracle %.2e" % (h, m, order, e))
        assert e < RTOL
    # the frames outside the paste ranges are the first take's, bit for bit
    first = b200mdm.stitch_handshake(W, ln, h, ms)
    lay = b200mdm.transition_layout(c["B"], c["T"], h, m, ln, ms)
    for k, (got, ft) in enumerate(zip(motions, first)):
        keep = torch.ones(ft.shape[-1], dtype=torch.bool)
        for i, (a, b) in enumerate(lay["paste"]):
            if lay["motion"][i] == k:
                keep[a:b] = False
        assert torch.equal(got.cpu()[..., keep], ft[..., keep])


# ------------------------------------------------------------------------------------------------ engine state
def test_engine_state_against_fresh_engines(small):
    cfg, diffusion, inp, y, shape, mask, motion = small
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    w = torch.rand(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    w2 = w.flip(-1).contiguous()
    ys = dict(soft=dict(y, inpainting_weight=w, inpainted_motion=motion), bool=dict(y, inpainting_mask=mask, inpainted_motion=motion),
              none=y, soft2=dict(y, inpainting_weight=w2, inpainted_motion=motion))
    for use_graph in (True, False):
        seq = ["soft", "bool", "none", "soft", "soft2"]   # soft2: only the weight differs from the loop before it
        got = [_run(diffusion, cfg, "ddim", shape, ys[k], xT, tape, use_graph) for k in seq]
        for k, v in zip(seq, got):
            fresh, d2 = _model(2, 6, 3)
            assert torch.equal(v, _run(d2, fresh, "ddim", shape, ys[k], xT, tape, use_graph)), (k, use_graph)
            fresh.model.engine().close()
    # b200mdm_set_cond clears the weight; b200mdm_denoise ignores it
    eng = cfg.model.engine()
    plain = _run(diffusion, cfg, "ddpm", shape, y, xT, tape, True)
    eng.set_cond(shape[0], shape[-1], y, True, "cuda")
    eng.set_inpaint_weight(w, motion)
    eng.set_cond(shape[0], shape[-1], y, True, "cuda")
    out = eng.sample_loop(_lib.MODE_DDPM, xT, tape, 0, _lib.FLAG_CLIP_DENOISED, True)
    torch.cuda.synchronize()
    assert torch.equal(out, plain)
    t = torch.full((shape[0],), 3, dtype=torch.long, device="cuda")
    bare = cfg(xT, t, y=y)
    eng.set_cond(shape[0], shape[-1], y, True, "cuda")
    eng.set_inpaint_weight(torch.ones(shape, device="cuda"), motion)
    assert torch.equal(eng.denoise(xT, t), bare)
