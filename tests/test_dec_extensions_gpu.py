"""GPU: the four sampling extensions on the BERT decoder with context_len 0 (humanml_trans_dec_512_bert):

  1. multi-prompt guidance: K = 1 with w = scale reproduces the reference's guided DDPM loop of this decoder
     (tests/golden/dip_longmem_small.npz, bert_ddpm: Mt = 100, ragged masks, T = 196) within 1e-3; K = 2 and 3 with
     prompts of different token counts (one over 64 tokens, the long cross-attention core) in every sampler family
     against the fp32 oracle (bert_dec_oracle.dec_denoiser) within 1e-3 * max(1, A / 4); permuting the prompts
     with their weights is bitwise invariant; zero weights give the unconditional forward exactly; the C ABI refuses
     b200mdm_set_cond_multi_tokens on DiP (ENOTIMPL) and CLIP-memory (EINVAL) engines;
  2. handshakes and refined transitions: windows against handshake_oracle.denoiser over the decoder oracle, h = 0 the
     plain loop bit for bit, refine_transitions against the DoubleTake oracle;
  3. joint-position control: zero weights are the unguided DDPM / DDIM loops bit for bit, guided loops match the oracle,
     the control loss does not increase;
  4. the headline shape (B = 64, T = 196, L = 8) for multi-prompt guidance at K = 2 and joint control;
  5. engine state: a plain CFG loop after each extension equals a fresh engine's bit for bit; Philox batch shards equal
     the whole batch bit for bit."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm import _lib, parallel
from b200mdm.engine import joint_guidance_hook
import bert_dec_oracle as bdo
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import double_take_oracle as dt
from oracle import dpm_oracle as dpo
from oracle import handshake_oracle as hso
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import reverse_oracle as ro
from oracle import ric_oracle
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3


def _bert(layers, steps, seed, ctx=0):
    """(model, diffusion, state dict) of a BERT decoder with synthetic weights (context_len ctx, 40 predicted frames)."""
    args = default_args(layers=layers, diffusion_steps=steps, arch="trans_dec", text_encoder_type="bert", context_len=ctx,
                        pred_len=40 if ctx else 0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=layers, cond_dim=768, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return model, diffusion, sd


def _prompt(B, Mt, seed, pad_from=None):
    """(tokens [Mt, B, 768], mask [B, Mt]) with sample 1 right-padded from pad_from."""
    enc, tmask, _ = b200mdm.synthetic_dip_inputs(B, Mt, 0, seed=seed)
    tmask[:] = False
    if pad_from is not None and B > 1:
        tmask[1, pad_from:] = True
    return enc, tmask


def _prompts(B, K, seed):
    """K prompts of 20, 70 (the long core) and 9 tokens."""
    sizes = [(20, 13), (70, 41), (9, None)]
    return [_prompt(B, Mt, seed + k, pad) for k, (Mt, pad) in enumerate(sizes[:K])]


def _cuda_pairs(pairs):
    return [(t.cuda(), m.cuda()) for t, m in pairs]


def _amp(w):
    return float(((1 - w.sum(1)).abs() + w.abs().sum(1)).max())


def _tol(w):
    return RTOL * max(1.0, _amp(w) / 4)


def _weights(case, B, K, T, g):
    if case == "body":
        up = b200mdm.body_part_mask("upper").float()[:, None]
        w = torch.stack([up, 1 - up], 0)[None].repeat(B, 1, 1, 1) * 2.5
        return w if K == 2 else torch.cat([w, torch.full((B, K - 2, 263, 1), 0.5)], 1)
    if case == "crossfade":
        t = torch.arange(T, dtype=torch.float32)
        a = ((t - T / 3) / (T / 3)).clamp(0, 1)
        w = torch.zeros(B, K, 1, T)
        w[:, 0, 0] = 2.5 * (1 - a)
        w[:, 1, 0] = 2.5 * a
        if K > 2:
            w[:, 2] = -1.0
        return w
    return torch.rand(B, K, 1, 1, generator=g) * 3 - 0.5


def _no_prefix(x):
    return x.new_zeros(x.shape[:-1] + (0,))


def _cfg_denoiser(W, enc, tmask, scale, lengths):
    """The guided decoder at schedule index i (the identity timestep map)."""
    return lambda x, i: mo.cfg_denoise_dec(W, x, i, enc, tmask, _no_prefix(x), scale, lengths)


# ------------------------------------------------------------------------------------------------ 1. multi-prompt
def test_k1_reproduces_reference_bert_golden(golden):
    from oracle import gen_golden_longmem as gl
    c = gl.BERT
    model, diffusion, _ = _bert(c["L"], c["steps"], c["weights_seed"])
    mp = b200mdm.MultiPromptSampleModel(model)
    inp, enc, tmask = gl.bert_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), prompt_embed=[(enc.cuda(), tmask.cuda())],
             prompt_weight=inp["scale"].view(c["B"], 1, 1, 1).cuda())
    out = diffusion.p_sample_loop(mp, (c["B"], 263, 1, c["T"]), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                  model_kwargs={"y": y}, noise_tape=torch.stack(inp["tape"][1:]).cuda())
    e = rel_err(out, golden("dip_longmem_small.npz")["bert_ddpm"])
    print("K=1 multi-prompt vs the reference's guided BERT decoder loop: %.3e" % e)
    assert e < RTOL


@pytest.mark.parametrize("K,case", [(2, "body"), (3, "crossfade"), (3, "scalars")])
def test_loops_vs_fp32_oracle(K, case):
    L, steps, B, T = 2, 6, 3, 24
    model, diffusion, sd = _bert(L, steps, 2)
    mp = b200mdm.MultiPromptSampleModel(model)
    g = torch.Generator().manual_seed(7 + K)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=13, lengths=[24, 15, 4])
    w = _weights(case, B, K, T, g)
    pairs = _prompts(B, K, 30)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), prompt_embed=_cuda_pairs(pairs), prompt_weight=w.cuda())
    f = bdo.dec_denoiser(mo.OracleWeights(sd, L), list(range(100)), pairs, w, inp["lengths"])
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    shape = (B, 263, 1, T)
    x, tape = inp["tape"][0], torch.stack(inp["tape"][1:])
    kw = dict(clip_denoised=False, model_kwargs={"y": y})
    res = {"ddpm": (diffusion.p_sample_loop(mp, shape, noise=x.cuda(), noise_tape=tape.cuda(), **kw),
                    deo.sample_loop(f, tabs, inp["tape"], "ddpm"))}
    for eta in (0.0, 0.5):
        res["ddim%g" % eta] = (diffusion.ddim_sample_loop(mp, shape, noise=x.cuda(), noise_tape=tape.cuda(), eta=eta, **kw),
                               deo.sample_loop(f, tabs, inp["tape"], "ddim", eta))
    res["plms"] = (diffusion.plms_sample_loop(mp, shape, noise=x.cuda(), order=2, **kw), po.plms_loop(f, tabs, x, order=2))
    res["dpm2m"] = (diffusion.dpm_solver_sample_loop(mp, shape, noise=x.cuda(), order=2, **kw), dpo.dpm_loop(f, tabs, x, order=2))
    res["inversion"] = (diffusion.ddim_reverse_sample_loop(mp, x.cuda(), **kw), ro.reverse_loop(f, tabs, x))
    tol = _tol(w)
    for k, (got, want) in res.items():
        e = rel_err(got, want)
        print("BERT decoder K=%d %-9s %-10s A=%.2f err %.3e (tol %.2e)" % (K, case, k, _amp(w), e, tol))
        assert e < tol, k


def test_permutation_zero_weights_and_c_abi_refusals():
    L, steps, B, T = 2, 4, 3, 24
    model, diffusion, _ = _bert(L, steps, 3)
    mp = b200mdm.MultiPromptSampleModel(model)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=11, lengths=[24, 17, 5])
    pairs = _cuda_pairs(_prompts(B, 3, 50))
    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda())
    x, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    # body-part weights on two prompts of 20 and 70 tokens with different padding: disjoint weights compose exactly in
    # either order, and the unconditional group's mask does not depend on the order
    wb = _weights("body", B, 2, T, None).cuda()
    run = lambda yy: diffusion.p_sample_loop(mp, x.shape, noise=x, clip_denoised=False, noise_tape=tape, model_kwargs={"y": yy})
    a = run(dict(base, prompt_embed=pairs[:2], prompt_weight=wb))
    b = run(dict(base, prompt_embed=pairs[1::-1], prompt_weight=wb.flip(1).contiguous()))
    assert torch.equal(a, b)
    # zero weights: the unconditional forward over the memory that admits every token some prompt admits
    t = torch.full((B,), 2, dtype=torch.long, device="cuda")
    tok, pad = model.engine().prompt_memories(pairs, B, "cuda")
    fu = model(x, t, y=dict(base, text_embed=(tok[0], torch.from_numpy(pad.min(0)).bool().cuda()), uncond=True))
    got = mp(x, t, y=dict(base, prompt_embed=pairs, prompt_weight=torch.zeros(B, 3, 1, 1, device="cuda")))
    assert torch.equal(got, fu)
    # the C ABI: prefix-completion engines ENOTIMPL, CLIP-memory engines EINVAL
    lib = _lib.load()
    tok = torch.zeros(1, 4, B, 768, device="cuda")
    mask = (ctypes.c_uint8 * (B * 4))()
    dip, _, _ = _bert(1, 4, 4, ctx=20)
    r = lib.b200mdm_set_cond_multi_tokens(dip.engine().h, B, 40, 1, ctypes.c_void_p(tok.data_ptr()), mask, 4, None, None)
    assert r == _lib.ENOTIMPL, r
    args = default_args(layers=1, diffusion_steps=4, arch="trans_dec", text_encoder_type="clip", emb_trans_dec=True)
    clip_dec, _ = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(clip_dec, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=1, cond_dim=512, seed=1))
    clip_dec.to("cuda").eval()
    r = lib.b200mdm_set_cond_multi_tokens(clip_dec.engine().h, B, 24, 1, ctypes.c_void_p(tok.data_ptr()), mask, 4, None, None)
    assert r == _lib.EINVAL, r
    # ... and the CLIP entry point on a BERT engine EINVAL
    r = lib.b200mdm_set_cond_multi_dec(model.engine().h, B, 24, 1, ctypes.c_void_p(tok.data_ptr()), None, None)
    assert r == _lib.EINVAL, r


# ------------------------------------------------------------------------------------------------ 2. handshake
@pytest.fixture(scope="module")
def windows():
    """5 windows of 40 frames in two motions, a 70-token memory with padding, guidance."""
    B, T, steps, L = 5, 40, 6, 2
    model, diffusion, sd = _bert(L, steps, 21)
    enc, tmask = _prompt(B, 70, 22, pad_from=33)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=23, lengths=[40, 36, 40, 40, 28],
                                   scale=torch.tensor([2.5, 1.0, 7.5, 2.5, 3.0]))
    ms = torch.tensor([True, False, False, True, False])
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             scale=inp["scale"].cuda(), motion_start=ms.cuda())
    return B, T, steps, L, model, diffusion, sd, enc, tmask, inp, ms, y


def test_handshake_windows_vs_oracle_and_h0(windows):
    B, T, steps, L, model, diffusion, sd, enc, tmask, inp, ms, y = windows
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    h = 4
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    den = hso.denoiser(_cfg_denoiser(W, enc, tmask, inp["scale"], inp["lengths"]), h, inp["lengths"], ms)
    kw = dict(noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": y})
    for name, fn, extra, sampler, eta in (("ddpm", diffusion.p_sample_loop, {}, "ddpm", 0.0),
                                          ("ddim", diffusion.ddim_sample_loop, {"eta": 0.0}, "ddim", 0.0)):
        got = fn(b200mdm.HandshakeSampleModel(cfg, h), (B, 263, 1, T), **kw, **extra)
        want = deo.sample_loop(den, tabs, inp["tape"], sampler, eta)
        e = rel_err(got, want)
        print("BERT decoder handshake h=%d %s: %.3e" % (h, name, e))
        assert e < RTOL
        plain = fn(cfg, (B, 263, 1, T), **kw, **extra)
        h0 = fn(b200mdm.HandshakeSampleModel(cfg, 0), (B, 263, 1, T), **kw, **extra)
        assert torch.equal(plain, h0), name


def test_refine_transitions_vs_double_take_oracle(windows):
    B, T, steps, L, model, diffusion, sd, enc, tmask, inp, ms, y = windows
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    h, m, k = 4, 3, 3
    ln = inp["lengths"]
    Wn = torch.randn(B, 263, 1, T, generator=torch.Generator().manual_seed(24)) * 0.5
    x_init = dt.gather(Wn, ln, ms, h, m)
    xT = torch.randn(x_init.shape, generator=torch.Generator().manual_seed(25))
    eps = torch.randn((steps - k,) + tuple(x_init.shape), generator=torch.Generator().manual_seed(26))
    motions = b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, Wn.cuda(), {"y": y}, h, m, k, noise=xT.cuda(),
                                         noise_tape=eps.cuda(), clip_denoised=False, eta=0.0)
    yt = bdo.transition_y(dict(text_embed=(enc, tmask), scale=inp["scale"]), ln, ms, h, m, x_init)
    te, tm = yt["text_embed"]
    W = mo.OracleWeights(sd, L)
    den = dt.denoiser(_cfg_denoiser(W, te, tm, yt["scale"], yt["lengths"]), yt["inpainting_weight"], x_init)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    with torch.no_grad():
        n = steps - k
        x = mo.q_sample(tabs, x_init, n - 1, xT)
        for j, i in enumerate(range(n - 1, -1, -1)):
            x = mo.ddim_step(tabs, den(x, i), x, i, eps[j])
    want = dt.paste(dt.stitch(Wn, ln, ms, h), x, ln, ms, h, m)
    for got, wm in zip(motions, want):
        e = rel_err(got, wm)
        print("BERT decoder refine_transitions h=%d m=%d: %.3e" % (h, m, e))
        assert e < RTOL


# ------------------------------------------------------------------------------------------------ 3. joint control
STEP, ITERS = 2e-4, 10


def _control(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    mean, std = jo.motion_stats(263)
    x = torch.randn(B, 263, T, generator=g) * 0.5
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    target = ric_oracle.recover_from_ric(data, 22).permute(0, 2, 3, 1).float()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    for j in (20, 21):
        weight[:, j, torch.arange(T // 4, T, max(1, T // 4))] = 1.0
    return mean, std, target, weight


def _weighted_error(sample, mean, std, target, weight):
    xyz = ric_oracle.sample_to_xyz(sample.cpu(), mean, std).double()
    return float((weight.double()[:, :, None] * (xyz - target.double()) ** 2).sum()) ** 0.5


def test_joint_control_zero_guided_and_loss(windows):
    B, T, steps, L, model, diffusion, sd, enc, tmask, inp, ms, y = windows
    y = {k: v for k, v in y.items() if k != "motion_start"}
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    mean, std, target, weight = _control(B, T, 5)
    jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    zero = dict(joint_target=target.cuda(), joint_weight=torch.zeros_like(weight).cuda())
    joint = dict(joint_target=target.cuda(), joint_weight=weight.cuda())
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = jo.guided_denoiser(_cfg_denoiser(W, enc, tmask, inp["scale"], inp["lengths"]), mean, std, target, weight, STEP, ITERS)
    shape = (B, 263, 1, T)
    for fn, extra, sampler in ((diffusion.p_sample_loop, {}, "ddpm"), (diffusion.ddim_sample_loop, {"eta": 0.0}, "ddim")):
        for use_graph in (True, False):
            plain = fn(cfg, shape, noise=xT, clip_denoised=False, noise_tape=tape, use_graph=use_graph,
                       model_kwargs={"y": y}, **extra)
            guided0 = fn(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape, use_graph=use_graph,
                         model_kwargs={"y": dict(y, **zero)}, **extra)
            assert torch.equal(plain, guided0), (sampler, use_graph)
        got = fn(jc, shape, noise=xT, clip_denoised=False, noise_tape=tape, model_kwargs={"y": dict(y, **joint)}, **extra)
        with torch.no_grad():
            want = deo.sample_loop(f, tabs, inp["tape"], sampler)
        e = rel_err(got, want)
        before, after = (_weighted_error(s, mean, std, target, weight) for s in (plain, got))
        print("BERT decoder joint control %s: vs oracle %.3e; weighted joint error %.4g -> %.4g" % (sampler, e, before, after))
        assert e < RTOL and after < before
    # the guidance iterations on this decoder's own x0: the control loss never increases
    t = torch.full((B,), steps - 1, dtype=torch.long, device="cuda")
    x0 = cfg(xT, t, y=y)
    _, loss = joint_guidance_hook(x0.reshape(B, 263, T), mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, ITERS)
    assert bool((loss[1:] <= loss[:-1] * (1 + 1e-6)).all())


# ------------------------------------------------------------------------------------------------ 4. headline shape
def test_headline_b64_multi_prompt_and_joint_control():
    L, steps, B, T, K = 8, 10, 64, 196, 2
    model, diffusion, sd = _bert(L, steps, 0)
    g = torch.Generator().manual_seed(1)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=2.5)
    pairs = [_prompt(B, 24, 60, pad_from=17), _prompt(B, 30, 61, pad_from=5)]
    w = _weights("crossfade", B, K, T, g)
    x, tape = inp["tape"][0], torch.stack(inp["tape"][1:])
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), prompt_embed=_cuda_pairs(pairs), prompt_weight=w.cuda())
    got = diffusion.ddim_sample_loop(b200mdm.MultiPromptSampleModel(model), (B, 263, 1, T), noise=x.cuda(),
                                     noise_tape=tape.cuda(), clip_denoised=False, model_kwargs={"y": y}).cpu()
    n = 3
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    f = bdo.dec_denoiser(W, list(range(steps)), [(t[:, :n], m[:n]) for t, m in pairs], w[:n], inp["lengths"][:n])
    with torch.no_grad():
        want = deo.sample_loop(f, tabs, [t[:n] for t in inp["tape"]], "ddim")
    e = rel_err(got[:n], want)
    print("B=64 T=196 L=8 BERT decoder DDIM %d steps, K=%d crossfade, 3 samples: %.3e" % (steps, K, e))
    assert e < _tol(w)
    enc, tmask = pairs[0]
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    mean, std, target, weight = _control(B, T, 8)
    yj = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
              scale=inp["scale"].cuda(), joint_target=target.cuda(), joint_weight=weight.cuda())
    got = diffusion.p_sample_loop(b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS), (B, 263, 1, T),
                                  noise=x.cuda(), noise_tape=tape.cuda(), clip_denoised=False, model_kwargs={"y": yj}).cpu()
    den = _cfg_denoiser(W, enc[:, :n], tmask[:n], inp["scale"][:n], inp["lengths"][:n])
    f = jo.guided_denoiser(den, mean, std, target[:n], weight[:n], STEP, ITERS)
    with torch.no_grad():
        want = deo.sample_loop(f, tabs, [t[:n] for t in inp["tape"]], "ddpm")
    e = rel_err(got[:n], want)
    print("B=64 T=196 L=8 BERT decoder DDPM %d steps, joint control, 3 samples: %.3e" % (steps, e))
    assert e < RTOL


# ------------------------------------------------------------------------------------------------ 5. engine state
def test_cfg_after_each_extension_equals_fresh_engine_and_philox_shards(windows):
    B, T, steps, L, model, diffusion, sd, enc, tmask, inp, ms, y = windows
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    shape = (B, 263, 1, T)
    ycfg = {k: v for k, v in y.items() if k != "motion_start"}
    mean, std, target, weight = _control(B, T, 9)
    pairs = _cuda_pairs(_prompts(B, 2, 70))
    wmp = _weights("crossfade", B, 2, T, None).cuda()
    ymp = dict(mask=y["mask"], lengths=y["lengths"], prompt_embed=pairs, prompt_weight=wmp)
    arms = {"handshake": (b200mdm.HandshakeSampleModel(cfg, 4), y),
            "joint": (b200mdm.JointControlSampleModel(cfg, mean, std, STEP, ITERS),
                      dict(ycfg, joint_target=target.cuda(), joint_weight=weight.cuda())),
            "multi": (b200mdm.MultiPromptSampleModel(model), ymp)}
    x = inp["tape"][0].cuda()
    fresh_model, _, _ = _bert(L, steps, 21)
    fresh = diffusion.p_sample_loop(b200mdm.ClassifierFreeSampleModel(fresh_model), shape, noise=x, clip_denoised=False,
                                    model_kwargs={"y": ycfg}, noise_seed=3)
    for name, (m, yy) in arms.items():
        diffusion.ddim_sample_loop(m, shape, noise=x, clip_denoised=False, model_kwargs={"y": yy}, noise_seed=3)
        after = diffusion.p_sample_loop(cfg, shape, noise=x, clip_denoised=False, model_kwargs={"y": ycfg}, noise_seed=3)
        assert torch.equal(after, fresh), name
    # Philox shards on motion boundaries (windows 0-2 and 3-4) equal the whole batch
    for name, (m, yy) in arms.items():
        full = diffusion.p_sample_loop(m, shape, clip_denoised=False, model_kwargs={"y": yy}, noise_seed=9)
        parts = [diffusion.p_sample_loop(m, (hi - lo,) + shape[1:], clip_denoised=False,
                                         model_kwargs=parallel.shard_model_kwargs({"y": yy}, lo, hi), noise_seed=9,
                                         sample_index_base=lo) for lo, hi in ((0, 3), (3, 5))]
        assert torch.equal(torch.cat(parts), full), name
