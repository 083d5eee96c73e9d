"""GPU: the variational bound (calc_bpd_loop) and p_mean_variance on the engine.

  * the EpiOut<OutVb> epilogue and its reduction alone (b200mdm_test_out_vb) bit for bit against a restatement fed with
    the engine's own x0 (torch on the GPU, in the kernel's operation and summation order), at i = n - 1, a middle index
    and i = 0, with and without the clamp and inpainting, FIXED_SMALL and FIXED_LARGE; mutants of the restatement
    (true and model mean swapped, the t = 0 thresholds one bin off, eps from the next row, the reduction without its
    last chunk) must differ;
  * calc_bpd_loop against every case of tests/golden/vb_small.npz (the unmodified reference): every column but t = 0
    within 1e-3; the t = 0 column against an fp64 restatement at the engine's x0 within a bound from its conditioning,
    and against the reference within 1e-2 bits;
  * the headline shape (B = 64, T = 196, 8 layers, guidance 2.5, 50 steps) against the fp32 oracle on 3 samples;
  * two runs, graph and eager (every kernel of the step under programmatic dependent launch), and torch's generator in
    chunks vs the same draws as a tape: identical bits; the Philox stream split over two batches equals one call;
    p_mean_variance's mean is the DDPM step's mean and q_posterior's mean of its pred_xstart; a bound loop between two
    sampling loops leaves the second one as a fresh engine computes it; a stale bound table is refused;
  * an unconstrained model and a model with a target against the fp32 oracle."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import gen_golden_vb as gv
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so
from oracle import vb_oracle as vo
from test_vb_cpu import golden_case

pytestmark = pytest.mark.gpu
RTOL = 1e-3
U = 2.0 ** -24
PRIOR_ABS = 2.0 ** -23 / math.log(2.0)


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _build(case):
    """(model the loop runs, diffusion, inputs, shape, y on the GPU) of a vb_small.npz case, on this project."""
    args, sdkw, num_actions, guided = gv.args_of(case)
    ds = SimpleNamespace(num_actions=num_actions) if num_actions else SimpleNamespace()
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=ds))
    if case == "respaced":
        diffusion = gv.gr.respaced_diffusion(gd, rs, gv.RESP)
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(**sdkw))
    model.to("cuda").eval()
    m = b200mdm.ClassifierFreeSampleModel(model) if guided else model
    inp, shape, extra = gv.inputs(case)
    y = gv.y_of(case, inp, extra, guided)
    y = {k: (tuple(t.cuda() for t in v) if isinstance(v, tuple) else v.cuda() if torch.is_tensor(v) else v) for k, v in y.items()}
    return m, diffusion, inp, shape, y


def _run(case, **kw):
    m, diffusion, inp, shape, y = _build(case)
    tape = torch.stack(inp["tape"][1:]).cuda()
    r = diffusion.calc_bpd_loop(m, inp["tape"][0].cuda(), clip_denoised=case == "enc_clip_inpaint", model_kwargs={"y": y},
                                noise_tape=tape, **kw)
    torch.cuda.synchronize()
    return r, (m, diffusion, inp, shape, y)


# ------------------------------------------------------------------------------------------------ the epilogue alone
def _split16(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def _x0_hook(lib, hres, scale, w, b, x, flags, mask, motion, B, JF, T, s_off, halves):
    out, pred = torch.empty_like(x), torch.empty_like(x)
    _lib.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w), _p(b), _p(x), None, None, _lib.MODE_X0, flags,
                                         _p(mask), _p(motion), _p(out), _p(pred), B, JF, T, 512, s_off, halves, _stream()))
    return pred


def _f(v):
    return torch.tensor(float(v), dtype=torch.float32, device="cuda")


def _restate(row, xs, xt, x0, nz, t0, row_eps=None, swap=False, lo=-0.999, hi=0.999):
    """The kernel's per-element terms in its fp32 operation order (torch CUDA ops: tanhf / logf as the kernel calls
    them); the keywords are the mutants."""
    c1, c2, lvt, lvm, sr, srm1 = (_f(row[k]) for k in range(6))
    klc, elv, isd = _f(row[8]), _f(row[9]), _f(row[10])
    if row_eps is not None:
        sr, srm1 = _f(row_eps[4]), _f(row_eps[5])
    mean = c1 * x0 + c2 * xt
    tm = c1 * xs + c2 * xt
    if swap:
        mean, tm = tm, mean
        klc = ((-1.0 + lvt) - lvm) + torch.exp(lvm - lvt)
        elv = torch.exp(-lvt)
    if t0:
        c = xs - mean

        def cdf(z):
            z3 = (z * z) * z
            return _f(0.5) * (_f(1.0) + torch.tanh(_f(np.float32(math.sqrt(2 / math.pi))) * (z + _f(0.044715) * z3)))
        cp = cdf(isd * (c + _f(np.float32(1 / 255))))
        cm = cdf(isd * (c - _f(np.float32(1 / 255))))
        lp = torch.where(xs < _f(lo), torch.log(cp.clamp(min=1e-12)),
                         torch.where(xs > _f(hi), torch.log((_f(1.0) - cm).clamp(min=1e-12)),
                                     torch.log((cp - cm).clamp(min=1e-12))))
        term = -lp
    else:
        d = tm - mean
        term = _f(0.5) * (klc + (d * d) * elv)
    dx = x0 - xs
    eps = (sr * xt - x0) / srm1
    de = eps - nz
    return term, dx * dx, de * de


def _means(elem, drop_last_chunk=False):
    return torch.stack([vo.engine_mean(elem[0].cpu(), True, drop_last_chunk), vo.engine_mean(elem[1].cpu(), False, drop_last_chunk),
                        vo.engine_mean(elem[2].cpu(), False, drop_last_chunk)])


@pytest.mark.parametrize("var", ["small", "large"])
@pytest.mark.parametrize("where", ["last", "middle", "zero"])
def test_epilogue_bit_exact(var, where):
    lib = _lib.load()
    d = rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(1000, "20"), betas=gd.get_named_beta_schedule("cosine", 1000),
                           model_mean_type=gd.ModelMeanType.START_X, loss_type=gd.LossType.MSE,
                           model_var_type=gd.ModelVarType.FIXED_SMALL if var == "small" else gd.ModelVarType.FIXED_LARGE)
    table = d.schedule_vb_rows()
    n = d.num_timesteps
    i = {"last": n - 1, "middle": 9, "zero": 0}[where]
    B, JF, T, s_off, halves = 3, 263, 40, 1, 2
    g = torch.Generator(device="cuda").manual_seed(31 + i)
    S = T + s_off
    hres = torch.cat(_split16(torch.randn(halves * B * S, 512, device="cuda", generator=g) * 1.2), 1).contiguous()
    scale = torch.tensor([1.0, 2.5, 7.5], device="cuda")
    w = torch.randn(JF, 512, device="cuda", generator=g) / 512 ** 0.5
    b = torch.randn(JF, device="cuda", generator=g) * 0.1
    xs = torch.randn(B, JF, T, device="cuda", generator=g)
    nz = torch.randn(B, JF, T, device="cuda", generator=g)
    row = torch.from_numpy(table[i]).cuda()
    xt = _f(table[i, 6]) * xs + _f(table[i, 7]) * nz
    for clip, inpaint in ((False, False), (True, False), (False, True), (True, True)):
        mask = (torch.rand(B, JF, T, device="cuda", generator=g) < 0.3).to(torch.uint8) if inpaint else None
        motion = torch.rand(B, JF, T, device="cuda", generator=g) * 2.4 - 1.2 if inpaint else None
        flags = _lib.FLAG_CLIP_DENOISED if clip else 0
        elem = torch.full((3, B, JF, T), float("nan"), device="cuda")
        terms = torch.full((3, B, n), -1.0, device="cuda")
        pred = torch.empty_like(xs)
        _lib.check(lib.b200mdm_test_out_vb(_p(hres), _p(scale), _p(w), _p(b), _p(xt), _p(xs), _p(nz), _p(row), i, n, flags,
                                           _p(mask), _p(motion), _p(pred), _p(elem), _p(terms), B, JF, T, 512, s_off, halves,
                                           _stream()))
        x0 = _x0_hook(lib, hres, scale, w, b, xt, flags, mask, motion, B, JF, T, s_off, halves)
        torch.cuda.synchronize()
        assert torch.equal(pred, x0)
        want = torch.stack(_restate(table[i], xs, xt, x0, nz, i == 0))
        assert torch.equal(elem, want), (clip, inpaint, (elem - want).abs().max())
        col = n - 1 - i
        got = terms[:, :, col].cpu()
        assert torch.equal(got, _means(want)), (clip, inpaint)
        others = torch.cat([terms[:, :, :col], terms[:, :, col + 1:]], 2)
        assert torch.all(others == -1.0)                                   # one column per step
        mutants = {"eps from the next row": _restate(table[i], xs, xt, x0, nz, i == 0, row_eps=table[(i + 1) % n])}
        if i == 0:
            mutants["model mean replaced by the true mean"] = _restate(table[i], xs, xt, x0, nz, True, swap=True)
            mutants["thresholds one bin off"] = _restate(table[i], xs, xt, x0, nz, True, lo=-0.999 + 2 / 255,
                                                         hi=0.999 - 2 / 255)
        elif table[i, 2] != table[i, 3]:
            mutants["true and model mean swapped"] = _restate(table[i], xs, xt, x0, nz, False, swap=True)
        for name, m in mutants.items():
            assert not torch.equal(_means(torch.stack(m)), got), name
        assert not torch.equal(_means(want, drop_last_chunk=True), got), "reduction missing the last chunk"


# ------------------------------------------------------------------------------------------------ parity
def _t0_bound(diffusion, xs, xt, x0):
    """(fp64 decoder term per sample in bits, a bound on its fp32 evaluation).  Per element, the clamped quantity q of
    the branch (cdf_plus, 1 - cdf_min or cdf_plus - cdf_min, each cdf in [0, 1]) is formed in fp32 with an absolute
    error of at most delta = 8u (2 + inv_std (|x| + |mean| + 1)) (the tanh and the rounded mean), so the fp32 term lies in
    [-log max(q + delta, 1e-12), -log max(q - delta, 1e-12)] up to the log's own 2u |log q|.  The bound is the distance
    from the fp64 term to the far end of that interval: delta / q where q is well above delta, at most
    log(q / 1e-12) + log(1 + delta / 1e-12) where the fp32 bin mass has cancelled."""
    xs, xt, x0 = xs.double().cpu(), xt.double().cpu(), x0.double().cpu()
    lvm = float(diffusion._model_log_variance()[0])
    mean = float(np.float32(diffusion.posterior_mean_coef1[0])) * x0 + float(np.float32(diffusion.posterior_mean_coef2[0])) * xt
    isd = math.exp(-0.5 * lvm)
    c = xs - mean
    cp = vo.approx_standard_normal_cdf(isd * (c + 1 / 255))
    cm = vo.approx_standard_normal_cdf(isd * (c - 1 / 255))
    q = torch.where(xs < -0.999, cp, torch.where(xs > 0.999, 1 - cm, cp - cm)).clamp(min=1e-12)
    nll = -torch.log(q)
    delta = 8 * U * (2 + isd * (xs.abs() + mean.abs() + 1))
    lo = -torch.log((q + delta).clamp(min=1e-12))
    hi = -torch.log((q - delta).clamp(min=1e-12))
    el = torch.maximum((nll - lo).abs(), (hi - nll).abs()) + 2 * U * nll.abs()
    B = xs.shape[0]
    return nll.reshape(B, -1).mean(1) / math.log(2), el.reshape(B, -1).mean(1) / math.log(2)


# |engine - reference| of the i = 0 column, in bits: both fp32, tanhf / logf on the GPU against torch's CPU tanh / log,
# whose ulp differences move cancelled bin masses; measured 9e-5 - 7.3e-3 bits over the seven cases (DESIGN.md section 2)
T0_ABS_BITS = 1e-2


@pytest.mark.parametrize("case", gv.CASES)
def test_parity_with_reference(case):
    r, (m, diffusion, inp, shape, y) = _run(case)
    want = golden_case(case)
    n = diffusion.num_timesteps
    for k in ("vb", "xstart_mse", "mse"):
        assert tuple(r[k].shape) == (shape[0], n)
    e = {k: rel_err(r[k].cpu(), want[k]) for k in ("xstart_mse", "mse")}
    e["vb t>0"] = rel_err(r["vb"][:, :-1].cpu(), want["vb"][:, :-1])
    print(case, " ".join("%s %.2e" % kv for kv in e.items()))
    assert max(e.values()) < RTOL, (case, e)
    # the prior is ~1e-5 bits at these schedules: 0.5 (prior_c + m^2) with prior_c = (-1 - lq) + exp(lq) cancelling to
    # ~lq^2 / 2; one ulp of prior_c (at 1: 2^-23) between torch's exp and numpy's is 2^-24 / log 2 bits of the mean
    perr = (r["prior_bpd"].cpu().double() - want["prior_bpd"].double()).abs()
    print(case, "prior: |engine - reference| %s" % perr.numpy())
    assert torch.all(perr <= RTOL * want["prior_bpd"].double().abs() + PRIOR_ABS), (case, perr)
    # t = 0: fp64 restatement at the engine's own x0 (p_mean_variance at the engine's x_t of that step)
    xs = inp["tape"][0].cuda()
    xt = _f(np.float32(diffusion.sqrt_alphas_cumprod[0])) * xs + _f(np.float32(diffusion.sqrt_one_minus_alphas_cumprod[0])) * inp["tape"][-1].cuda()
    t = torch.zeros(shape[0], dtype=torch.long, device="cuda")
    x0 = diffusion.p_mean_variance(m, xt, t, clip_denoised=case == "enc_clip_inpaint", model_kwargs={"y": y})["pred_xstart"]
    f64, bound = _t0_bound(diffusion, xs, xt, x0)
    err = (r["vb"][:, -1].cpu().double() - f64).abs()
    ref_err = (want["vb"][:, -1].double() - r["vb"][:, -1].cpu().double()).abs()
    print(case, "t=0: |engine - fp64| %s, bound %s, |reference - engine| %s" % (err.numpy(), bound.numpy(), ref_err.numpy()))
    assert torch.all(err <= bound), (case, err, bound)
    assert torch.all(ref_err <= T0_ABS_BITS), (case, ref_err)
    # total_bpd: n fp32 additions in column order, then the prior
    tot = r["vb"].cpu().double().sum(1) + r["prior_bpd"].cpu().double()
    tb = (n + 1) * U * (r["vb"].cpu().double().abs().sum(1) + r["prior_bpd"].cpu().double().abs())
    assert torch.all((r["total_bpd"].cpu().double() - tot).abs() <= tb)
    assert rel_err(r["total_bpd"].cpu(), want["total_bpd"]) < RTOL


def test_headline_shape():
    L, steps, B, T = 8, 50, 64, 196
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=L, diffusion_steps=steps),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=L, seed=0)
    b200mdm.load_model_wo_clip(model, sd)
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=10, scale=torch.full((B,), 2.5),
                                   lengths=[T - 3 * (b % 40) for b in range(B)])
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    tape = torch.stack(inp["tape"][1:]).cuda()
    r = diffusion.calc_bpd_loop(cfg, inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    torch.cuda.synchronize()
    S = 3
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    W = mo.OracleWeights(sd, L)
    f = po.enc_denoiser(W, list(range(steps)), inp["text_embed"][:, :S], inp["scale"][:S], inp["lengths"][:S])
    with torch.no_grad():
        o = vo.vb_loop(f, tabs, inp["tape"][0][:S], [e[:S] for e in inp["tape"][1:]], False)
    e = {k: rel_err(r[k][:S].cpu(), o[k]) for k in ("xstart_mse", "mse", "prior_bpd")}
    e["vb t>0"] = rel_err(r["vb"][:S, :-1].cpu(), o["vb"][:, :-1])
    e["total_bpd"] = rel_err(r["total_bpd"][:S].cpu(), o["total_bpd"])
    print("headline:", " ".join("%s %.2e" % kv for kv in e.items()))
    assert max(e.values()) < RTOL, e


# ------------------------------------------------------------------------------------------------ determinism, noise
def test_deterministic_graph_and_generator():
    case = "enc_cfg"
    r1, (m, diffusion, inp, shape, y) = _run(case)
    r2, _ = _run(case)
    xs = inp["tape"][0].cuda()
    tape = torch.stack(inp["tape"][1:]).cuda()
    r3 = diffusion.calc_bpd_loop(m, xs, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape, use_graph=False)
    diffusion.NOISE_CHUNK = 3                                 # the generator path in three chunks
    torch.manual_seed(123)
    r4 = diffusion.calc_bpd_loop(m, xs, clip_denoised=False, model_kwargs={"y": y})
    torch.manual_seed(123)
    drawn = torch.stack([torch.randn_like(xs) for _ in range(diffusion.num_timesteps)])
    r5 = diffusion.calc_bpd_loop(m, xs, clip_denoised=False, model_kwargs={"y": y}, noise_tape=drawn)
    torch.cuda.synchronize()
    for k in gv.KEYS:
        print(k, "runs", torch.equal(r1[k], r2[k]), "graph/eager", torch.equal(r1[k], r3[k]),
              float((r1[k] - r3[k]).abs().max()), "generator", torch.equal(r4[k], r5[k]))
    for k in gv.KEYS:
        assert torch.equal(r1[k], r2[k]) and torch.equal(r1[k], r3[k]), k
        assert torch.equal(r4[k], r5[k]), k


def test_philox_batch_split():
    case = "enc_cfg"
    m, diffusion, inp, shape, y = _build(case)
    xs = inp["tape"][0].cuda()
    whole = diffusion.calc_bpd_loop(m, xs, clip_denoised=False, model_kwargs={"y": y}, noise_seed=77)
    parts = []
    for lo, hi in ((0, 1), (1, 3)):
        yp = dict(mask=y["mask"][lo:hi], lengths=y["lengths"][lo:hi], text_embed=y["text_embed"][:, lo:hi],
                  scale=y["scale"][lo:hi])
        parts.append(diffusion.calc_bpd_loop(m, xs[lo:hi].contiguous(), clip_denoised=False, model_kwargs={"y": yp},
                                             noise_seed=77, sample_index_base=lo))
    torch.cuda.synchronize()
    for k in gv.KEYS:
        assert torch.equal(whole[k], torch.cat([p[k] for p in parts])), k
    other = diffusion.calc_bpd_loop(m, xs, clip_denoised=False, model_kwargs={"y": y}, noise_seed=78)
    assert not torch.equal(other["vb"], whole["vb"])


def test_p_mean_variance_is_the_ddpm_mean():
    m, diffusion, inp, shape, y = _build("enc_clip_inpaint")
    x = inp["tape"][1].cuda()
    for i in (0, 3, diffusion.num_timesteps - 1):
        t = torch.full((shape[0],), i, dtype=torch.long, device="cuda")
        for clip in (False, True):
            out = diffusion.p_mean_variance(m, x, t, clip_denoised=clip, model_kwargs={"y": y})
            step = diffusion.p_sample(m, x, t, clip_denoised=clip, model_kwargs={"y": y}, noise=torch.zeros_like(x))
            torch.cuda.synchronize()
            assert torch.equal(out["mean"], step["sample"]) and torch.equal(out["pred_xstart"], step["pred_xstart"])
            # and, independently of the step, q_posterior's mean of the returned x0 in fp32 from the fp64 tables
            want = (_f(np.float32(diffusion.posterior_mean_coef1[i])) * out["pred_xstart"]
                    + _f(np.float32(diffusion.posterior_mean_coef2[i])) * x)
            assert torch.equal(out["mean"], want), (i, clip)
            assert torch.equal(out["log_variance"].cpu()[:, 0, 0, 0],
                               torch.full((shape[0],), float(np.float32(diffusion.posterior_log_variance_clipped[i]))))
            assert out["variance"].shape == x.shape
    with pytest.raises(AssertionError):
        diffusion.p_mean_variance(m, x, torch.tensor([1, 2, 2], device="cuda"), model_kwargs={"y": y})


def test_engine_state_and_stale_table():
    case = "enc_cfg"
    m, diffusion, inp, shape, y = _build(case)
    noise = inp["tape"][1].cuda()
    tape = torch.stack(inp["tape"][1:]).cuda()
    a = diffusion.p_sample_loop(m, shape, noise=noise, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    diffusion.calc_bpd_loop(m, inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    b = diffusion.p_sample_loop(m, shape, noise=noise, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    m2, d2, _, _, y2 = _build(case)
    fresh = d2.p_sample_loop(m2, shape, noise=noise, clip_denoised=False, model_kwargs={"y": y2}, noise_tape=tape)
    torch.cuda.synchronize()
    assert torch.equal(a, fresh) and torch.equal(b, fresh)
    eng = m.model.engine() if hasattr(m, "model") else m.engine()
    eng.set_schedule(diffusion.schedule_rows(0.0), list(range(diffusion.num_timesteps)))   # the bound table goes stale
    terms = torch.empty(3, shape[0], diffusion.num_timesteps, device="cuda")
    with pytest.raises(Exception, match="set_schedule_vb"):
        eng.vb_loop_range(diffusion.num_timesteps - 1, 1, inp["tape"][0].cuda(), tape, 0, terms, None)
    with pytest.raises(Exception, match="continue"):
        eng2 = m2.model.engine()
        eng2.set_schedule_vb(d2.schedule_vb_rows())
        eng2.set_cond(shape[0], shape[-1], y2, True, "cuda")
        eng2.vb_loop_range(diffusion.num_timesteps - 1, 1, None, tape, 0, terms, None)


# ------------------------------------------------------------------------------------------------ other model kinds
JOINTS = b200mdm.synthetic.HML_TARGET_JOINTS


@pytest.mark.parametrize("kind", ["unconstrained", "target"])
def test_other_model_kinds_vs_oracle(kind):
    """An unconstrained model (no conditioning, no CFG) and text + a single-MLP target with CFG, 6 steps, against the
    fp32 oracle: every vb column but i = 0, the mse tables and total_bpd within 1e-3."""
    from oracle import target_oracle as to
    L, steps, B, T = 2, 6, 3, 24
    over = dict(layers=L, diffusion_steps=steps)
    if kind == "unconstrained":
        over["unconstrained"] = True
        sd = b200mdm.synthetic_state_dict(num_layers=L, seed=21, cond_mode="no_cond")
    else:
        over.update(multi_target_cond=True, multi_encoder_type="single", target_enc_layers=1)
        sd = b200mdm.synthetic_state_dict(num_layers=L, seed=22, target_encoder="single")
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=23, lengths=[24, 17, 5],
                                   scale=torch.tensor([2.5, 1.0, 7.5]))
    W = mo.OracleWeights(sd, L)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda())
    if kind == "unconstrained":
        m = model

        def f(x, i):
            return mo.denoise_enc(W, x, i, None, inp["lengths"])
    else:
        m = b200mdm.ClassifierFreeSampleModel(model)
        tg = b200mdm.synthetic_target_inputs(B, seed=24)
        y.update(text_embed=inp["text_embed"].cuda(), scale=inp["scale"].cuda(), target_cond=tg["target_cond"].cuda(),
                 target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
        gt = to.target_embedding(W, "single", tg["target_cond"], to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"]))

        def f(x, i):
            return to.cfg(to.denoise_enc, inp["scale"], W, x, i, inp["text_embed"], gt, inp["lengths"])
    tape = torch.stack(inp["tape"][1:]).cuda()
    r = diffusion.calc_bpd_loop(m, inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    torch.cuda.synchronize()
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    with torch.no_grad():
        o = vo.vb_loop(f, tabs, inp["tape"][0], inp["tape"][1:], False)
    e = {k: rel_err(r[k].cpu(), o[k]) for k in ("xstart_mse", "mse", "total_bpd")}
    e["vb t>0"] = rel_err(r["vb"][:, :-1].cpu(), o["vb"][:, :-1])
    print(kind, " ".join("%s %.2e" % kv for kv in e.items()))
    assert max(e.values()) < RTOL, (kind, e)
