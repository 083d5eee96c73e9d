"""GPU: multistep DPM-Solver++ (dpm_solver_sample_loop / dpm_solver_sample_loop_progressive).

  * the EpiOut<OutDpm> epilogue alone (b200mdm_test_out_dpm) bit for bit against an unfused fp32 restatement of the
    documented update, at orders 1 and 2, at the first step, a middle index and i = 0, with and without the clamp and
    inpainting; four mutants of the restatement must differ;
  * order 1 against the unmodified reference's DDIM eta = 0 samples (tests/golden/enc_small.npz, dec_emb_small.npz)
    within 1e-3, and against the engine's own DDIM eta = 0 loop on the same x_T within a measured rounding bound;
  * order 2 against oracle/dpm_oracle.py on the fp32 model oracles, 1e-3 relative on every step: trans_enc text with
    CFG, clamp + inpainting, a2m unguided, DiP through AutoRegressiveSampler, the CLIP decoder with a timestep token, and
    the c2 shape (B = 64, T = 196, L = 8, 20 steps respaced from 1000) per sample;
  * graph and eager runs, B200MDM_PDL=0 and the default, a loop split into two range calls, a batch split into halves
    and the progressive form are bit-identical to the loop."""
import importlib
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import dpm_oracle as do
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
# ||DPM order 1 - DDIM eta 0||_F / ||DDIM||_F on the engine, same x_T, 20 steps respaced from 1000: the same step in two
# fp32 forms.  DDIM's eps = (sr*x - x0)/srm1 cancels at the noisy end (sr ~ 2e4 at the last index); the DPM form
# c_x*x + c0*x0 does not.  Measured on an H100 (DESIGN.md section 2); the bound is the project's parity tolerance
SELF_DDIM_BOUND = 1e-3
deo = importlib.import_module("oracle.dec_emb_oracle")
syn = importlib.import_module("motion-diffusion-model_b200.synthetic")


def _spaced(steps, respacing):
    return rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(steps, respacing),
                              betas=gd.get_named_beta_schedule("cosine", steps), model_mean_type=gd.ModelMeanType.START_X,
                              model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)


def _enc(layers, steps, seed, guided=True, respacing=None, **over):
    """(sampled model, model, diffusion, state dict); `respacing`: the diffusion keeps those steps of `steps`."""
    args = default_args(layers=layers, diffusion_steps=steps, **over)
    ds = {"num_actions": 12} if over.get("dataset") == "humanact12" else {}
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace(**ds)))
    if respacing is not None:
        diffusion = _spaced(steps, respacing)
    kw = dict(input_feats=150, cond_mode="action", num_actions=12) if over.get("dataset") == "humanact12" else {}
    if over.get("multi_target_cond"):
        kw["target_encoder"] = over["multi_encoder_type"]
    sd = b200mdm.synthetic_state_dict(num_layers=layers, seed=seed, **kw)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), model, diffusion, sd


def _y(inp, scale=True, **extra):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(), **extra)
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _steps(diffusion, m, shape, x, y, order=2, clip=False):
    """Every step's sample (progressive form); the loop equals the last one bit for bit."""
    prog = [o["sample"] for o in diffusion.dpm_solver_sample_loop_progressive(m, shape, noise=x, clip_denoised=clip,
                                                                              model_kwargs={"y": y}, order=order)]
    loop = diffusion.dpm_solver_sample_loop(m, shape, noise=x, clip_denoised=clip, model_kwargs={"y": y}, order=order)
    assert torch.equal(loop, prog[-1])
    return prog


def _vs_oracle(name, steps, denoise, tables, x, order=2, clip=False, inpaint=None):
    ref = []
    do.dpm_loop(denoise, tables, x, order=order, clip_denoised=clip, inpaint=inpaint, collect=ref)
    assert len(steps) == len(ref)
    errs = [rel_err(s, r) for s, (r, _) in zip(steps, ref)]
    print("%s: relative error per step vs the fp32 oracle %s" % (name, " ".join("%.2e" % e for e in errs)))
    assert max(errs) < RTOL, (name, errs)


# ------------------------------------------------------------------------------------------------ the epilogue alone
def _split16(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _x0_hook(lib, hres, scale, w, b, x, flags, mask, motion, B, JF, T, s_off, halves):
    """x0 as the DDIM epilogue forms it (b200mdm_test_out_step, mode X0): CFG blend, projection, inpainting, clamp."""
    out, pred = torch.empty_like(x), torch.empty_like(x)
    _lib.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w), _p(b), _p(x), None, None, _lib.MODE_X0, flags,
                                         _p(mask), _p(motion), _p(out), _p(pred), B, JF, T, 512, s_off, halves, _stream()))
    return pred


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("where", ["first", "start", "middle", "last"])
def test_epilogue_bit_exact(order, where):
    """first: step 0 at i = n - 1; start: step 0 of a loop that starts at a middle index (skip_timesteps); middle: a
    second-order step; last: i = 0."""
    lib = _lib.load()
    d = _spaced(1000, "20")
    table = d.schedule_dpm_rows()
    n = d.num_timesteps
    i, k = {"first": (n - 1, 0), "start": (9, 0), "middle": (9, 10), "last": (0, n - 1)}[where]
    B, JF, T, s_off, halves = 4, 263, 40, 1, 2
    g = torch.Generator(device="cuda").manual_seed(17 * order + i)
    S = T + s_off
    h = torch.randn(halves * B * S, 512, device="cuda", generator=g) * 1.2
    hres = torch.cat(_split16(h), 1).contiguous()
    scale = torch.tensor([0.0, 1.0, 2.5, 7.5], device="cuda")
    w = torch.randn(JF, 512, device="cuda", generator=g) / 512 ** 0.5
    b = torch.randn(JF, device="cuda", generator=g) * 0.1
    x = torch.randn(B, JF, T, device="cuda", generator=g)
    row = torch.from_numpy(table[i]).cuda()
    for clip, inpaint in ((False, False), (True, False), (False, True), (True, True)):
        mask = (torch.rand(B, JF, T, device="cuda", generator=g) < 0.3).to(torch.uint8) if inpaint else None
        motion = torch.rand(B, JF, T, device="cuda", generator=g) * 2.4 - 1.2 if inpaint else None
        flags = _lib.FLAG_CLIP_DENOISED if clip else 0
        hist = torch.randn(2, B, JF, T, device="cuda", generator=g)
        x0_prev = hist[(k - 1) % 2].clone()
        untouched = hist[(k - 1) % 2].clone()
        out = torch.full_like(x, float("nan"))
        _lib.check(lib.b200mdm_test_out_dpm(_p(hres), _p(scale), _p(w), _p(b), _p(x), _p(row), i, k, order, flags,
                                            _p(mask), _p(motion), _p(hist), _p(out), B, JF, T, 512, s_off, halves,
                                            _stream()))
        x0 = _x0_hook(lib, hres, scale, w, b, x, flags, mask, motion, B, JF, T, s_off, halves)
        raw = _x0_hook(lib, hres, scale, w, b, x, 0, None, None, B, JF, T, s_off, halves)
        torch.cuda.synchronize()
        assert torch.equal(hist[k % 2], x0), (clip, inpaint)             # the history keeps the x0 the update uses
        assert torch.equal(hist[(k - 1) % 2], untouched)
        xn, x0n, x0pn, r = x.cpu().numpy(), x0.cpu().numpy(), x0_prev.cpu().numpy(), table[i]
        second = order == 2 and k > 0 and i > 0
        want = do.update32(r, xn, x0n, x0pn if second else None)
        got = out.cpu().numpy()
        assert np.array_equal(got, want), (clip, inpaint, np.abs(got - want).max())
        if i == 0:
            assert np.array_equal(got, x0n)                               # the last step returns x0 exactly
        mutants = {"c_cur and c_prev swapped": do.update32(r[[0, 1, 3, 2]], xn, x0n, x0pn)}
        if second:
            mutants["history read from slot k"] = do.update32(r, xn, x0n, hist[k % 2].cpu().numpy())
        if k == 0 and i == n - 1:
            assert r[3] == 0 and r[2] == r[1]        # no previous step: the row itself is first order
        elif k == 0:
            mutants["first step at second order"] = do.update32(r, xn, x0n, x0pn)
        if inpaint or clip:
            mutants["x0 before inpainting / clamp in the history"] = raw.cpu().numpy()
            assert not torch.equal(hist[k % 2], raw)
        if second or k == 0:
            for name, m in mutants.items():
                if name.startswith("x0 before"):
                    continue
                assert not np.array_equal(got, m), name


# ------------------------------------------------------------------------------------------------ anchors
def test_order1_vs_reference_ddim_eta0(golden):
    """enc_small: L=2, 4 steps, CFG (2.5, 1.0, 7.5) -- the unmodified reference's ddim_sample_loop at eta = 0."""
    g = golden("enc_small.npz")
    cfg, _, diffusion, _ = _enc(2, 4, 1)
    inp = b200mdm.synthetic_inputs(3, nframes=24, steps=4, seed=11, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 7.5]))
    x = inp["tape"][0].cuda()
    out = diffusion.dpm_solver_sample_loop(cfg, (3, 263, 1, 24), noise=x, clip_denoised=False, model_kwargs={"y": _y(inp)},
                                           order=1)
    e = rel_err(out, g["ddim_eta0"])
    print("order 1 vs the reference's DDIM eta 0 (enc_small): %.2e" % e)
    assert e < RTOL

    g = golden("dec_emb_small.npz")
    args = default_args(layers=2, diffusion_steps=4, arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, syn.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=512, seed=9))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(3, nframes=24, steps=4, seed=15, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 7.5]))
    out = diffusion.dpm_solver_sample_loop(cfg, (3, 263, 1, 24), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                           model_kwargs={"y": _y(inp)}, order=1)
    e = rel_err(out, g["ddim_eta0"])
    print("order 1 vs the reference's DDIM eta 0 (dec_emb_small): %.2e" % e)
    assert e < RTOL


def test_order1_vs_engine_ddim_eta0():
    """The engine's own DDIM eta = 0 loop on the same x_T, for every model kind: text CFG, a2m, a target, clamp +
    inpainting, at 20 steps respaced from 1000."""
    cases = []
    cfg, _, diffusion, _ = _enc(2, 1000, 3, respacing="20")
    inp = b200mdm.synthetic_inputs(4, nframes=60, steps=0, seed=21, lengths=[60, 41, 20, 3],
                                   scale=torch.tensor([2.5, 1.0, 2.5, 0.0]))
    cases.append(("text CFG", cfg, diffusion, (4, 263, 1, 60), inp["tape"][0], _y(inp), False))
    motion = torch.rand(4, 263, 1, 60) * 1.8 - 0.9
    imask = torch.zeros(4, 263, 1, 60, dtype=torch.bool)
    imask[..., :12] = True
    cases.append(("clamp + inpainting", cfg, diffusion, (4, 263, 1, 60), inp["tape"][0],
                  _y(inp, inpainting_mask=imask.cuda(), inpainted_motion=motion.cuda()), True))
    model, _, diffusion_a, _ = _enc(2, 1000, 4, guided=False, respacing="20", dataset="humanact12", cond_mask_prob=0.0)
    ia = b200mdm.synthetic_inputs(3, njoints=25, nfeats=6, nframes=60, steps=0, seed=22, lengths=[60, 45, 30])
    cases.append(("a2m", model, diffusion_a, (3, 25, 6, 60), ia["tape"][0],
                  dict(mask=ia["mask"].cuda(), lengths=ia["lengths"].cuda(), action=torch.tensor([[3], [11], [0]]).cuda()),
                  False))
    cfg_t, _, diffusion_t, _ = _enc(2, 1000, 5, respacing="20", multi_target_cond=True, multi_encoder_type="single",
                                    target_enc_layers=1)
    tg = syn.synthetic_target_inputs(4, seed=5)
    cases.append(("target", cfg_t, diffusion_t, (4, 263, 1, 60), inp["tape"][0],
                  _y(inp, target_cond=tg["target_cond"].cuda(), target_joint_names=tg["target_joint_names"],
                     is_heading=tg["is_heading"]), False))
    for name, m, dif, shape, x, y, clip in cases:
        kw = dict(noise=x.cuda(), clip_denoised=clip, model_kwargs={"y": y})
        dpm = dif.dpm_solver_sample_loop(m, shape, order=1, **kw)
        ddim = dif.ddim_sample_loop(m, shape, eta=0.0, noise_seed=1, **kw)
        e = rel_err(dpm, ddim)
        print("order 1 vs the engine's DDIM eta 0 (%s): %.2e" % (name, e))
        assert e < SELF_DDIM_BOUND, (name, e)
        o2 = dif.dpm_solver_sample_loop(m, shape, order=2, **kw)
        assert torch.isfinite(o2).all() and not torch.equal(o2, dpm)


# ------------------------------------------------------------------------------------------------ end to end, order 2
def test_enc_text_cfg_and_inpainting_vs_oracle():
    cfg, _, diffusion, sd = _enc(2, 8, 6)
    inp = b200mdm.synthetic_inputs(3, nframes=24, steps=0, seed=23, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 2.0]))
    W = mo.OracleWeights(sd, 2)
    f = po.enc_denoiser(W, list(range(8)), inp["text_embed"], inp["scale"], inp["lengths"])
    tabs = so.diffusion_tables(so.named_betas("cosine", 8))
    x, shape = inp["tape"][0], (3, 263, 1, 24)
    _vs_oracle("text CFG", _steps(diffusion, cfg, shape, x.cuda(), _y(inp)), f, tabs, x)
    motion = torch.rand(shape, generator=torch.Generator().manual_seed(4)) * 1.8 - 0.9
    imask = torch.zeros(shape, dtype=torch.bool)
    imask[..., :8] = True
    y = _y(inp, inpainting_mask=imask.cuda(), inpainted_motion=motion.cuda())
    _vs_oracle("clamp + inpainting", _steps(diffusion, cfg, shape, x.cuda(), y, clip=True), f, tabs, x, clip=True,
               inpaint=(imask, motion))


def test_a2m_unguided_vs_oracle():
    model, _, diffusion, sd = _enc(2, 6, 2, guided=False, dataset="humanact12", cond_mask_prob=0.0)
    inp = b200mdm.synthetic_inputs(4, njoints=25, nfeats=6, nframes=60, steps=0, seed=12, lengths=[60, 60, 45, 30])
    action = torch.tensor([[3], [11], [0], [5]])
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), action=action.cuda())
    W = mo.OracleWeights(sd, 2)
    f = lambda x, i: mo.denoise_enc(W, x, i, None, inp["lengths"], True, False, action)
    x = inp["tape"][0]
    _vs_oracle("a2m", _steps(diffusion, model, (4, 25, 6, 60), x.cuda(), y), f,
               so.diffusion_tables(so.named_betas("cosine", 6)), x)


def test_clip_decoder_vs_oracle():
    L, steps, B, T = 2, 6, 3, 24
    args = default_args(layers=L, diffusion_steps=steps, arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=9)
    b200mdm.load_model_wo_clip(model, sd)
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=15, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 2.0]))
    f = deo.denoiser(mo.OracleWeights(sd, L), list(range(steps)), inp["text_embed"], inp["scale"], inp["lengths"])
    x = inp["tape"][0]
    _vs_oracle("CLIP decoder", _steps(diffusion, cfg, (B, 263, 1, T), x.cuda(), _y(inp)), f,
               so.diffusion_tables(so.named_betas("cosine", steps)), x)


def test_dip_autoregressive_vs_oracle():
    """DiP (Mt = 16) through AutoRegressiveSampler: 2 chunks of 40 frames, the prefix handed from chunk to chunk."""
    B, ctx, pred, Mt, steps, need = 2, 20, 40, 16, 5, 80
    args = default_args(layers=2, diffusion_steps=steps, arch="trans_dec", text_encoder_type="bert", context_len=ctx,
                        pred_len=pred)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=22)
    b200mdm.load_model_wo_clip(model, sd)
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    W = mo.OracleWeights(sd, 2)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, ctx, seed=33)
    scale = torch.tensor([2.5, 1.0])
    chunks = [b200mdm.synthetic_inputs(B, nframes=pred, steps=0, seed=40 + i, scale=scale) for i in range(2)]
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    cur, buf = prefix, []
    for c in chunks:
        f = po.dec_denoiser(W, list(range(steps)), enc, tmask, cur, scale, c["lengths"])
        s = do.dpm_loop(f, tabs, c["tape"][0], order=2)
        buf.append(s)
        cur = s[..., -ctx:]
    want = torch.cat(buf, -1)[..., :need]
    y = dict(mask=chunks[0]["mask"].cuda(), lengths=chunks[0]["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             prefix=prefix.cuda(), scale=scale.cuda())
    sampler = b200mdm.AutoRegressiveSampler(args, diffusion.dpm_solver_sample_loop, required_frames=need)
    out = sampler.sample(cfg, (B, 263, 1, need), clip_denoised=False, model_kwargs={"y": y},
                         noise=torch.stack([c["tape"][0] for c in chunks]).cuda())
    e = rel_err(out, want)
    print("DiP through AutoRegressiveSampler, order 2: %.2e" % e)
    assert out.shape == (B, 263, 1, need) and e < RTOL


def test_c2_shape_20_steps_vs_oracle():
    B, T, L = 64, 196, 8
    cfg, _, diffusion, sd = _enc(L, 1000, 0, respacing="20")
    assert diffusion.num_timesteps == 20
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    x = inp["tape"][0]
    out = diffusion.dpm_solver_sample_loop(cfg, (B, 263, 1, T), noise=x.cuda(), clip_denoised=False,
                                           model_kwargs={"y": _y(inp)})
    assert torch.isfinite(out).all()
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(np.asarray(so.respaced(so.named_betas("cosine", 1000),
                                                      so.space_timesteps(1000, "20"))[0]))
    for b in (0, 31, 63):
        f = po.enc_denoiser(W, diffusion.timestep_map, inp["text_embed"][:, [b]], inp["scale"][[b]], inp["lengths"][[b]])
        ref = do.dpm_loop(f, tabs, x[[b]], order=2)
        e = rel_err(out[[b]], ref)
        print("c2 shape, 20 steps, sample %d: %.2e" % (b, e))
        assert e < RTOL, (b, e)


# ------------------------------------------------------------------------------------------------ bit identity
def test_graph_eager_split_halves_progressive_identical():
    cfg, _, diffusion, _ = _enc(2, 1000, 7, respacing="12")
    B, shape = 4, (4, 263, 1, 40)
    inp = b200mdm.synthetic_inputs(B, nframes=40, steps=0, seed=31, lengths=[40, 33, 12, 2],
                                   scale=torch.tensor([2.5, 1.0, 2.0, 0.0]))
    x = inp["tape"][0].cuda()
    y = _y(inp)
    kw = dict(noise=x, clip_denoised=True, model_kwargs={"y": y})
    for order in (1, 2):
        ref = diffusion.dpm_solver_sample_loop(cfg, shape, order=order, **kw)
        assert torch.equal(ref, diffusion.dpm_solver_sample_loop(cfg, shape, order=order, use_graph=False, **kw))
        prog = list(diffusion.dpm_solver_sample_loop_progressive(cfg, shape, order=order, **kw))
        assert len(prog) == 12 and torch.equal(prog[-1]["sample"], ref)
        assert torch.equal(prog[-1]["pred_xstart"], ref)                   # the last step returns x0
        eager = list(diffusion.dpm_solver_sample_loop_progressive(cfg, shape, order=order, use_graph=False, **kw))
        assert all(torch.equal(a["sample"], b["sample"]) and torch.equal(a["pred_xstart"], b["pred_xstart"])
                   for a, b in zip(prog, eager))
        # one loop split into two range calls
        eng = cfg.model.engine()
        out = torch.empty_like(x)
        for use_graph in (True, False):
            eng.dpm_loop_range(order, 11, 5, x, None, 2, use_graph)
            eng.dpm_loop_range(order, 6, 7, None, out, 2, use_graph)
            torch.cuda.synchronize()
            assert torch.equal(out, ref), (order, use_graph)
        # a batch split into halves equals the whole batch
        halves = []
        for lo, hi in ((0, 2), (2, 4)):
            yh = dict(mask=y["mask"][lo:hi], lengths=y["lengths"][lo:hi], text_embed=y["text_embed"][:, lo:hi],
                      scale=y["scale"][lo:hi])
            halves.append(diffusion.dpm_solver_sample_loop(cfg, (2,) + shape[1:], noise=x[lo:hi], clip_denoised=True,
                                                           model_kwargs={"y": yh}, order=order))
        assert torch.equal(torch.cat(halves), ref), order
    # continuation of a different order, a stale table and a table of the wrong length are refused
    eng = cfg.model.engine()
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.dpm_loop_range(1, 3, 1, None, None, 0, True)
    assert exc.value.code == _lib.ESTATE
    n = diffusion.num_timesteps
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.set_schedule_dpm(np.zeros((n + 1, 4), dtype=np.float32))
    assert exc.value.code == _lib.EINVAL
    eng.set_schedule(diffusion.schedule_rows(0.0), diffusion.timestep_map)
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.dpm_loop_range(2, n - 1, n, x, None, 0, True)
    assert exc.value.code == _lib.ESTATE
    again = diffusion.dpm_solver_sample_loop(cfg, shape, order=2, **kw)        # _dpm_begin sets the table again
    assert torch.equal(again, diffusion.dpm_solver_sample_loop(cfg, shape, order=2, use_graph=False, **kw))


_PDL_SCRIPT = r"""
import sys, torch, numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from types import SimpleNamespace
import b200mdm
from conftest import default_args
model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=2, diffusion_steps=10),
                                                      SimpleNamespace(dataset=SimpleNamespace()))
b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=2, seed=8))
cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
inp = b200mdm.synthetic_inputs(3, nframes=30, steps=0, seed=9, scale=torch.tensor([2.5, 1.0, 2.0]))
y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(), scale=inp["scale"].cuda())
out = diffusion.dpm_solver_sample_loop(cfg, (3, 263, 1, 30), noise=inp["tape"][0].cuda(), model_kwargs={"y": y})
np.save(sys.argv[2], out.cpu().numpy())
"""


def test_pdl_off_is_bit_identical(tmp_path):
    outs = []
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for pdl in ("0", None):
        env = dict(os.environ)
        env.pop("B200MDM_PDL", None)
        if pdl is not None:
            env["B200MDM_PDL"] = pdl
        path = str(tmp_path / ("pdl%s.npy" % pdl))
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _PDL_SCRIPT, root, path]
        subprocess.run(cmd, check=True, env=env, cwd=root)
        outs.append(np.load(path))
    assert np.array_equal(outs[0], outs[1])
