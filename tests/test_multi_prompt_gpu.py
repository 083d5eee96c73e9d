"""GPU: multi-prompt guidance (MultiPromptSampleModel; compose_step_kernel, DESIGN.md "Multi-prompt guidance").

  1. anchored to the reference: K = 1 with w = y['scale'] reproduces the reference's own CFG forwards and loops
     (tests/golden/enc_small.npz, dec_emb_small.npz) within 1e-3;
  2. routing: upper / lower body masks of weight 1 give M x0_A + (1 - M) x0_B of the engine's own single-prompt
     forwards; zero weights give the unconditional forward; permuting the prompts with their weight rows leaves the
     sample bitwise unchanged;
  3. loops against the fp32 oracle (oracle/multi_prompt_oracle.py) within 1e-3 * max(1, A / 4), A = |1 - sum w| +
     sum |w| the error amplification of the composition: DDPM, DDIM at eta 0 and 0.5, PLMS, DPM-Solver++ 2M and DDIM
     inversion at K = 2 and 3 for the encoder, the CLIP decoder and an action model, with body-part, crossfade and
     negative-prompt weights, inpainting and target conditioning; one headline-shape case (B = 64, T = 196, L = 8);
  4. engine state: a composed loop followed by a CFG loop equals a fresh engine's CFG loop bit for bit; Philox shards
     equal the 1-GPU result bit for bit; the ENOTIMPL refusals of the C ABI."""
import importlib
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import dpm_oracle as dpo
from oracle import mdm_oracle as mo
from oracle import multi_prompt_oracle as mpo
from oracle import plms_oracle as po
from oracle import reverse_oracle as ro
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3
syn = importlib.import_module("motion-diffusion-model_b200.synthetic")


def _build(kind, layers, steps, seed, **over):
    """(model, diffusion, state dict, feature count) of a trans_enc CLIP ('enc'), CLIP-decoder ('dec') or action
    ('a2m') model with synthetic weights."""
    data = SimpleNamespace()
    if kind == "dec":
        over = dict(arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True, **over)
        sd_kw = dict(arch="trans_dec", cond_dim=512,
                     target_encoder=over.get("multi_encoder_type") if over.get("multi_target_cond") else None)
    elif kind == "a2m":
        over = dict(dataset="humanact12", **over)
        data = SimpleNamespace(num_actions=12)
        sd_kw = dict(input_feats=150, cond_mode="action", num_actions=12)
    else:
        sd_kw = {}
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=layers, diffusion_steps=steps, **over),
                                                          SimpleNamespace(dataset=data))
    sd = syn.synthetic_state_dict(num_layers=layers, seed=seed, **sd_kw)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return model, diffusion, sd, 150 if kind == "a2m" else 263


def _amp(w):
    """max over elements of A = |1 - sum_k w_k| + sum_k |w_k|"""
    return float(((1 - w.sum(1)).abs() + w.abs().sum(1)).max())


def _tol(w):
    return RTOL * max(1.0, _amp(w) / 4)


def _weights(case, B, K, D, T, g):
    """[B, K, D or 1, T or 1] weights of a named case."""
    if case == "body":                               # upper body from prompt 0, lower body from prompt 1 (D = 263)
        up = b200mdm.body_part_mask("upper").float()[:, None]
        w = torch.stack([up, 1 - up], 0)[None].repeat(B, 1, 1, 1) * 2.5
        return w if K == 2 else torch.cat([w, torch.full((B, K - 2, D, 1), 0.5)], 1)
    if case == "crossfade":                          # prompt 0 -> prompt 1 over the middle third, prompt 2 negative
        t = torch.arange(T, dtype=torch.float32)
        a = ((t - T / 3) / (T / 3)).clamp(0, 1)
        w = torch.zeros(B, K, 1, T)
        w[:, 0, 0] = 2.5 * (1 - a)
        w[:, 1, 0] = 2.5 * a
        if K > 2:
            w[:, 2] = -1.0
        return w
    return (torch.rand(B, K, 1, 1, generator=g) * 3 - 0.5)          # per-motion scalars, some negative


def _y(inp, K, w, dev="cuda", g=None, **extra):
    B = inp["text_embed"].shape[1]
    pe = torch.randn(K, B, 512, generator=g) * 0.5 if g is not None else inp["text_embed"].expand(K, B, 512)
    return dict(mask=inp["mask"].to(dev), lengths=inp["lengths"].to(dev), prompt_embed=pe.to(dev), prompt_weight=w.to(dev),
                **extra)


# ------------------------------------------------------------------------------------------------ 1. the reference
def test_k1_reproduces_reference_cfg_golden(golden):
    B, T = 3, 24
    shape = (B, 263, 1, T)
    t = torch.full((B,), 2, dtype=torch.long, device="cuda")
    for kind, name, seed, inp_seed in (("enc", "enc_small.npz", 1, 11), ("dec", "dec_emb_small.npz", 9, 15)):
        g = golden(name)
        model, diffusion, _, _ = _build(kind, 2, 4, seed)
        mp = b200mdm.MultiPromptSampleModel(model)
        inp = b200mdm.synthetic_inputs(B, nframes=T, steps=4, seed=inp_seed, lengths=[24, 17, 5],
                                       scale=torch.tensor([2.5, 1.0, 7.5]))
        w = inp["scale"].view(B, 1, 1, 1)
        x, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
        kw = dict(noise=x, clip_denoised=False, noise_tape=tape)
        got = {"fwd_cfg": mp(x, t, y=_y(inp, 1, w)),
               "ddim_eta0": diffusion.ddim_sample_loop(mp, shape, eta=0.0, model_kwargs={"y": _y(inp, 1, w)}, **kw)}
        ddpm = diffusion.p_sample_loop(mp, shape, model_kwargs={"y": _y(inp, 1, w)}, **kw)
        if kind == "enc":
            got["ddpm_steps"] = ddpm
            want = dict(g, ddpm_steps=golden("enc_small_steps.npz")["ddpm_steps"][-1])
        else:
            got["ddpm"] = ddpm
            want = g
        motion = torch.from_numpy(g["inpaint_motion"]).cuda()
        m = torch.zeros(shape, dtype=torch.bool, device="cuda")
        m[..., :8] = True
        got["ddpm_inpaint"] = diffusion.p_sample_loop(mp, shape, model_kwargs={
            "y": _y(inp, 1, w, inpainting_mask=m, inpainted_motion=motion)}, **kw)
        for k, v in got.items():
            e = rel_err(v, want[k])
            print("%s %-12s %.3e" % (kind, k, e))
            assert e < RTOL, (kind, k)


# ------------------------------------------------------------------------------------------------ 2. routing
def test_routing_body_masks_zero_weights_and_permutation():
    B, T = 3, 24
    model, diffusion, _, _ = _build("enc", 2, 4, 1)
    mp = b200mdm.MultiPromptSampleModel(model)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=4, seed=11, lengths=[24, 17, 5])
    g = torch.Generator().manual_seed(5)
    pe = torch.randn(2, B, 512, generator=g) * 0.5
    x = inp["tape"][0].cuda()
    t = torch.full((B,), 2, dtype=torch.long, device="cuda")
    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda())
    fa = model(x, t, y=dict(base, text_embed=pe[:1].cuda()))
    fb = model(x, t, y=dict(base, text_embed=pe[1:].cuda()))
    fu = model(x, t, y=dict(base, text_embed=pe[:1].cuda(), uncond=True))
    M = b200mdm.body_part_mask("upper").float().view(1, 263, 1, 1).cuda()
    w = torch.stack([M.view(263, 1), 1 - M.view(263, 1)], 0)[None].repeat(B, 1, 1, 1)
    y = dict(base, prompt_embed=pe.cuda(), prompt_weight=w)
    got = mp(x, t, y=y)
    e = rel_err(got, M * fa + (1 - M) * fb)
    print("body routing vs single-prompt forwards: %.3e" % e)
    assert e < 1e-5
    e = rel_err(mp(x, t, y=dict(y, prompt_weight=torch.zeros(B, 2, 1, 1, device="cuda"))), fu)
    print("zero weights vs the unconditional forward: %.3e" % e)
    assert e < 1e-5
    shape = (B, 263, 1, T)
    tape = torch.stack(inp["tape"][1:]).cuda()
    wb = _weights("body", B, 2, 263, T, g).cuda()
    run = lambda yy: diffusion.p_sample_loop(mp, shape, noise=x, clip_denoised=False, noise_tape=tape, model_kwargs={"y": yy})
    a = run(dict(base, prompt_embed=pe.cuda(), prompt_weight=wb))
    b = run(dict(base, prompt_embed=pe.flip(0).cuda(), prompt_weight=wb.flip(1).contiguous()))
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ 3. loops vs the oracle
def _oracle_denoiser(kind, W, K, y, inp, w, g_target=None):
    ln = inp["lengths"]
    if kind == "a2m":
        return mpo.enc_denoiser(W, list(range(100)), None, w, ln, actions=y["prompt_action"].cpu())
    if kind == "dec":
        return mpo.dec_emb_denoiser(W, list(range(100)), y["prompt_embed"].cpu(), w, ln, g=g_target)
    return mpo.enc_denoiser(W, list(range(100)), y["prompt_embed"].cpu(), w, ln)


@pytest.mark.parametrize("kind,K,case", [("enc", 2, "body"), ("enc", 3, "crossfade"), ("dec", 3, "body"),
                                         ("dec", 2, "crossfade"), ("a2m", 2, "scalars"), ("a2m", 3, "crossfade")])
def test_loops_vs_fp32_oracle(kind, K, case):
    L, steps, B, T = 2, 6, 3, 24
    model, diffusion, sd, D = _build(kind, L, steps, 2)
    mp = b200mdm.MultiPromptSampleModel(model)
    g = torch.Generator().manual_seed(7 + K)
    J, Fe = (25, 6) if kind == "a2m" else (263, 1)
    inp = b200mdm.synthetic_inputs(B, njoints=J, nfeats=Fe, nframes=T, steps=steps, seed=13, lengths=[24, 15, 4])
    w = _weights(case, B, K, D, T, g)
    y = _y(inp, K, w, g=g)
    if kind == "a2m":
        y.pop("prompt_embed")
        y["prompt_action"] = torch.randint(0, 12, (B, K), generator=g)
    W = mo.OracleWeights(sd, L)
    f = _oracle_denoiser(kind, W, K, y, inp, w)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    shape = (B, J, Fe, T)
    x, tape = inp["tape"][0], torch.stack(inp["tape"][1:])
    tol = _tol(w)
    kw = dict(clip_denoised=False, model_kwargs={"y": y})
    res = {}
    res["ddpm"] = (diffusion.p_sample_loop(mp, shape, noise=x.cuda(), noise_tape=tape.cuda(), **kw),
                   deo.sample_loop(f, tabs, inp["tape"], "ddpm"))
    for eta in (0.0, 0.5):
        res["ddim%g" % eta] = (diffusion.ddim_sample_loop(mp, shape, noise=x.cuda(), noise_tape=tape.cuda(), eta=eta, **kw),
                               deo.sample_loop(f, tabs, inp["tape"], "ddim", eta))
    res["plms"] = (diffusion.plms_sample_loop(mp, shape, noise=x.cuda(), order=2, **kw), po.plms_loop(f, tabs, x, order=2))
    res["dpm2m"] = (diffusion.dpm_solver_sample_loop(mp, shape, noise=x.cuda(), order=2, **kw), dpo.dpm_loop(f, tabs, x, order=2))
    res["inversion"] = (diffusion.ddim_reverse_sample_loop(mp, x.cuda(), **kw), ro.reverse_loop(f, tabs, x))
    m = torch.zeros(shape, dtype=torch.bool)
    m[..., :6] = True
    motion = torch.randn(shape, generator=g) * 0.5
    yi = dict(y, inpainting_mask=m.cuda(), inpainted_motion=motion.cuda())
    res["ddpm_inpaint"] = (diffusion.p_sample_loop(mp, shape, noise=x.cuda(), noise_tape=tape.cuda(), clip_denoised=False,
                                                   model_kwargs={"y": yi}),
                           deo.sample_loop(f, tabs, inp["tape"], "ddpm", inpaint=(m, motion)))
    for k, (got, want) in res.items():
        e = rel_err(got, want)
        print("%s K=%d %-9s %-12s A=%.2f err %.3e (tol %.2e)" % (kind, K, case, k, _amp(w), e, tol))
        assert e < tol, k


def test_target_conditioning_vs_fp32_oracle():
    L, steps, B, T, K = 2, 6, 3, 24, 2
    model, diffusion, sd, _ = _build("dec", L, steps, 9, multi_target_cond=True, multi_encoder_type="single",
                                     target_enc_layers=1)
    mp = b200mdm.MultiPromptSampleModel(model)
    g = torch.Generator().manual_seed(3)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=15, lengths=[24, 17, 5])
    tg = syn.synthetic_target_inputs(B, seed=5)
    ty = dict(target_cond=tg["target_cond"].cuda(), target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    w = _weights("crossfade", B, K, 263, T, g)
    y = _y(inp, K, w, g=g, **ty)
    gt = model.engine().test_target(ty["target_cond"], _valid(model, ty, B)).cpu()
    W = mo.OracleWeights(sd, L)
    f = mpo.dec_emb_denoiser(W, list(range(steps)), y["prompt_embed"].cpu(), w, inp["lengths"], g=gt)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    got = diffusion.p_sample_loop(mp, (B, 263, 1, T), noise=inp["tape"][0].cuda(), noise_tape=torch.stack(inp["tape"][1:]).cuda(),
                                  clip_denoised=False, model_kwargs={"y": y})
    e = rel_err(got, deo.sample_loop(f, tabs, inp["tape"], "ddpm"))
    print("target conditioning, DDPM: %.3e" % e)
    assert e < _tol(w)


def _valid(model, ty, B):
    from b200mdm.engine import canonical_target
    return canonical_target(ty, B, model.engine().target_joint_names)[1]


def test_headline_shape_vs_fp32_oracle():
    L, steps, B, T, K = 8, 10, 64, 196, 2
    model, diffusion, sd, _ = _build("enc", L, steps, 0)
    mp = b200mdm.MultiPromptSampleModel(model)
    g = torch.Generator().manual_seed(1)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10)
    w = _weights("crossfade", B, K, 263, T, g)
    y = _y(inp, K, w, g=g)
    x, tape = inp["tape"][0], torch.stack(inp["tape"][1:])
    got = diffusion.ddim_sample_loop(mp, (B, 263, 1, T), noise=x.cuda(), noise_tape=tape.cuda(), clip_denoised=False,
                                     model_kwargs={"y": y}).cpu()
    n = 3
    f = mpo.enc_denoiser(mo.OracleWeights(sd, L), list(range(steps)), y["prompt_embed"][:, :n].cpu(), w[:n],
                         inp["lengths"][:n])
    want = deo.sample_loop(f, so.diffusion_tables(so.named_betas("cosine", steps)), [t[:n] for t in inp["tape"]], "ddim")
    e = rel_err(got[:n], want)
    print("B=64 T=196 L=8 DDIM %d steps, K=%d crossfade, 3 samples: %.3e" % (steps, K, e))
    assert e < _tol(w)


# ------------------------------------------------------------------------------------------------ 4. engine state
def test_composed_then_cfg_equals_fresh_engine_and_philox_shards():
    B, T, steps = 4, 30, 5
    model, diffusion, sd, _ = _build("enc", 2, steps, 4)
    mp, cfg = b200mdm.MultiPromptSampleModel(model), b200mdm.ClassifierFreeSampleModel(model)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=17, lengths=[30, 22, 9, 1], scale=torch.tensor([2.5, 1.0, 3.0, 0.5]))
    g = torch.Generator().manual_seed(2)
    shape = (B, 263, 1, T)
    ycfg = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
                scale=inp["scale"].cuda())
    ymp = _y(inp, 3, _weights("crossfade", B, 3, 263, T, g), g=g)
    x = inp["tape"][0].cuda()
    for use_graph in (True, False):
        diffusion.ddim_sample_loop(mp, shape, noise=x, clip_denoised=False, model_kwargs={"y": ymp}, noise_seed=3,
                                   use_graph=use_graph)
        after = diffusion.p_sample_loop(cfg, shape, noise=x, clip_denoised=False, model_kwargs={"y": ycfg}, noise_seed=3,
                                        use_graph=use_graph)
        fresh_model, _, _, _ = _build("enc", 2, steps, 4)
        fresh = diffusion.p_sample_loop(b200mdm.ClassifierFreeSampleModel(fresh_model), shape, noise=x, clip_denoised=False,
                                        model_kwargs={"y": ycfg}, noise_seed=3, use_graph=use_graph)
        assert torch.equal(after, fresh), use_graph
    full = diffusion.p_sample_loop(mp, shape, clip_denoised=False, model_kwargs={"y": ymp}, noise_seed=9)
    parts = [diffusion.p_sample_loop(mp, (hi - lo,) + shape[1:], clip_denoised=False,
                                     model_kwargs=parallel.shard_model_kwargs({"y": ymp}, lo, hi), noise_seed=9,
                                     sample_index_base=lo) for lo, hi in ((0, 1), (1, 4))]
    assert torch.equal(torch.cat(parts), full)


def test_enotimpl_refusals():
    B, T = 2, 16
    model, diffusion, _, _ = _build("enc", 1, 4, 4)
    eng = model.engine()
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=1, seed=1)
    w = torch.ones(B, 2, 1, 1, device="cuda")
    y = _y(inp, 2, w, g=torch.Generator().manual_seed(0))
    eng.set_cond_multi(B, T, y, y["prompt_embed"], None, w, "cuda")
    with pytest.raises(_lib.B200MDMError) as ei:
        eng.set_handshake(2, B, T, {})
    assert ei.value.code == _lib.ENOTIMPL
    with pytest.raises(_lib.B200MDMError) as ei:
        eng.set_joint_guidance(torch.zeros(263, device="cuda"), torch.ones(263, device="cuda"),
                               torch.zeros(B, 22, 3, T, device="cuda"), torch.ones(B, 22, T, device="cuda"), 1e-3, 2)
    assert ei.value.code == _lib.ENOTIMPL
    import ctypes
    lib = _lib.load()
    # the bound loop (its table armed first: a missing table is ESTATE before the refusal)
    eng.set_schedule(diffusion.schedule_rows(0.0), diffusion._timestep_map(), key=None)
    eng.set_schedule_vb(diffusion.schedule_vb_rows())
    x = torch.zeros(B, 263, 1, T, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.b200mdm_vb_loop_range(eng.h, 3, 4, ctypes.c_void_p(x.data_ptr()), None, 0, _lib.FLAG_PHILOX_NOISE, None, None,
                                     1, s) == _lib.ENOTIMPL
    assert b"multi-prompt guidance" in lib.b200mdm_last_error()
    assert lib.b200mdm_set_prompt_weight(eng.h, 3, ctypes.c_void_p(w.data_ptr()), 0, 0, 0, 0, None) == _lib.EINVAL
    assert lib.b200mdm_set_prompt_weight(eng.h, 2, ctypes.c_void_p(w.data_ptr()), -1, 0, 0, 0, None) == _lib.EINVAL
    eng.set_cond(B, T, dict(text_embed=inp["text_embed"].cuda()), False, "cuda")      # clears the composition
    assert lib.b200mdm_set_prompt_weight(eng.h, 2, ctypes.c_void_p(w.data_ptr()), 0, 0, 0, 0, None) == _lib.ESTATE
