"""GPU: the guided DDPM / DDIM step against its guidance hook, step by step (DESIGN.md, "Joint-position control",
"The guided step").

The guided step runs the forward of b200mdm_denoise, with the MODE_X0 output GEMM writing the step's x0 into the
workspace's jg_x0, then joint_guidance_step_kernel: the guidance iterations of the test hooks (joint_guidance_run) and
the output step's tail (inpainting, the clamp of clip_denoised, the update).  Both sides are fp32 with explicit
round-to-nearest operations, so for one step

    pred_xstart == clamp(inpaint(hook(denoise(x_t, t))))      and      sample == update(pred_xstart, x_t, noise, row i)

bit for bit, where denoise is the wrapper's plain call and hook the b200mdm_test_{joint,foot,scene}_guidance kernel
the engine's descriptor selects, fed the case's targets, weights, lambda, K, contacts, lengths, grids and floor.  The
inputs that differ between the two sides are exactly the engine's wiring: the descriptor upload, jg_x0, the sample a
CTA reads, the lengths staging, the grids' per-sample strides, the kernel variant and the order of the tail.

  a. one step of each case of tests/guided_step_cases.py (trans_enc with scales 0 / 1 / 2.5 / 7.5 and ragged lengths,
     KIT, the CLIP decoder with a timestep token, the BERT decoder at T = 256; T = 1 and 2; first, middle and last
     schedule index; joint, joint + foot, foot with given contacts, scene with a shared curved SDF and per-sample
     terrains, and the reverse; clip_denoised, bool and soft inpainting; the headline shape B = 64, T = 196, L = 8 per
     feature set): p_sample / ddim_sample and Engine.sample_step against the expectation, and the hook against the
     fp64 oracle within 2^-12 max |dx| + 2 u K max |x0| (its loss within 2^-16 G_0; planar grids only);
  b. every step of DDPM, DDIM eta 0 and 0.5 _progressive loops with a noise tape, the graph and eager loops' last
     sample, and a Philox loop against the step-by-step chain;
  c. mutants: each wiring mistake of guided_step_cases.mutants (and, in b, the raw x0 of the next step) differs from
     the engine's bits and misses the fp64 bound at least 8-fold (printed);
  d. a captured step graph follows a new lambda and K, targets in another tensor, targets edited in place and new
     grids; a sequence of feature sets on one engine equals fresh engines; two workspaces alternate; the kernel count
     of a guided step."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.engine import foot_guidance_hook, joint_guidance_hook, scene_guidance_hook
import guided_step_cases as gc
from test_epilogues_gpu import _step_f32, check_x_out

pytestmark = pytest.mark.gpu
MODE = {"ddpm": _lib.MODE_DDPM, "ddim": _lib.MODE_DDIM}


def _model(c):
    args, sdkw = gc.model_args(c)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(**sdkw)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), diffusion


def _jc(cfg, k, **over):
    kw = dict(gc.wrapper_kw(k), **over)
    step, iters = kw.pop("step", k.step), kw.pop("iters", k.iters)
    return b200mdm.JointControlSampleModel(cfg, k.mean, k.std, step, iters, **kw)


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _t(k, i):
    return torch.full((k.B,), i, dtype=torch.long, device="cuda")


def hook(k, x0, g):
    """(guided x0 [n, D, 1, T], loss [K + 1, n]) of x0 [n, D, 1, T] by the test hook of the terms g switches on"""
    n = x0.shape[0]
    x = x0.reshape(n, k.D, k.T)
    dev = lambda t: None if t is None else t.cuda()   # noqa: E731
    a = (x, k.mean.cuda(), k.std.cuda(), g["target"].cuda(), g["weight"].cuda(), g["step"], g["iters"])
    if g["scene"]:
        out, loss = scene_guidance_hook(*a, k.cw, k.fw, k.fh, k.ow, k.r, g["sdf"], g["terrain"], dev(g["contact"]),
                                        g["lengths"])
    elif g["foot"]:
        out, loss = foot_guidance_hook(*a, k.cw, k.fw, k.fh, dev(g["contact"]), g["lengths"])
    else:
        out, loss = joint_guidance_hook(*a)
    return out.reshape(x0.shape), loss


def expected(k, x0, g, order=None):
    """(pred_xstart, the hook's guided x0, its loss) of the step's x0 [B, D, 1, T] in tail order `order`"""
    rows = list(range(k.B))
    if order == "after_inpaint":
        h, loss = hook(k, gc.inpaint(k, x0, rows), g)
        return gc.clamp(k, h), h, loss
    if order == "after_clamp":
        h, loss = hook(k, gc.clamp(k, gc.inpaint(k, x0, rows)), g)
        return h, h, loss
    h, loss = hook(k, x0, g)
    return gc.clamp(k, gc.inpaint(k, h, rows)), h, loss


def check_update(mode, row, pred, x_t, noise, sample, i):
    """sample bit for bit against the float32 update of pred (check_x_out; at i = 0 the update is x0 itself, where an
    FMA-contracted evaluation cannot differ)"""
    if i != 0:
        check_x_out(mode, pred, x_t, noise, sample, row=row)
        return
    want = _step_f32(mode, pred.cpu().numpy(), x_t.cpu().numpy(), noise.cpu().numpy(), row)
    assert np.array_equal(sample.cpu().numpy().view(np.int32), want.view(np.int32))
    assert _bits_equal(sample, pred)


def check_fp64(k, x0, h, loss, label):
    """the hook's guided x0 and loss of motions k.idx against the fp64 oracle: (fp64 pred_xstart, bound)"""
    rows = k.idx
    x0c = x0[rows].cpu()
    want, want_loss = gc.guide64(k, x0c, gc.guide_inputs(k))
    bnd = gc.bound(k, x0c, want, k.iters)
    err = float((h[rows].cpu().double().reshape(want.shape) - want).abs().max())
    lsub = loss[:, rows].cpu().double()
    lerr = float(((lsub - want_loss).abs() / (gc.EPS_L * want_loss[0].clamp_min(1e-30))).max())
    print("%s: |dx| %.3g, hook err / bound %.3f, loss err / bound %.3f"
          % (label, float((want - x0c.double().reshape(want.shape)).abs().max()), err / bnd, lerr))
    assert err <= bnd and lerr <= 1.0, label
    return gc.clamp(k, gc.inpaint(k, want, rows, True)), bnd


def check_mutants(k, x0, x0_cond, pred, pred64, bnd, label, planar):
    """every mutant differs from the engine's pred bits and, with planar grids, misses the fp64 bound 8-fold"""
    rows = list(range(k.B))
    for m, (g, src, order) in gc.mutants(k, rows).items():
        mut, _, _ = expected(k, x0_cond if src == "cond" else x0, g, order)
        assert not _bits_equal(mut, pred), (label, m)
        miss = float((mut[k.idx].cpu().double().reshape(pred64.shape) - pred64).abs().max()) / bnd
        print("   mutant %-20s misses the bound %.1f-fold" % (m, miss))
        if planar:
            assert miss >= gc.MISS, (label, m, miss)


def one_step(k, cfg, diffusion, sampler, eta, i, label, fp64=True, mutants=True):
    """(a) and (c) for schedule index i of case k"""
    jc = _jc(cfg, k)
    eng = cfg.model.engine()
    y = gc.y_dict(k, "cuda")
    x_t, noise = k.xt.cuda(), k.noise.cuda()
    mode = MODE[sampler]
    fn = diffusion.p_sample if sampler == "ddpm" else diffusion.ddim_sample
    kw = {} if sampler == "ddpm" else {"eta": eta}
    out = fn(jc, x_t, _t(k, i), clip_denoised=k.clip, model_kwargs={"y": y}, noise=noise, **kw)
    flags = _lib.FLAG_CLIP_DENOISED if k.clip else 0
    s2, p2 = eng.sample_step(mode, i, x_t, noise, flags, want_pred=True)      # the engine as the sampler left it
    x0 = jc(x_t, _t(k, i), y=gc.y_dict(k, "cuda"))                           # b200mdm_denoise: the plain model
    pred, h, loss = expected(k, x0, gc.guide_inputs(k, list(range(k.B))))
    ok = _bits_equal(pred, out["pred_xstart"]), _bits_equal(pred, p2), _bits_equal(out["sample"], s2)
    print("%s %s eta %.1f i %d: pred_xstart == tail(hook(denoise)) %s, Engine.sample_step pred %s, sample %s"
          % (label, sampler, eta, i, ok[0], ok[1], ok[2]))
    assert all(ok), label
    check_update(mode, diffusion.schedule_rows(eta)[i], pred, x_t, noise, out["sample"], i)
    if not fp64:
        return
    planar = k.sdf is None or not k.c["feat"].endswith("shared_sdf")
    if planar:
        pred64, bnd = check_fp64(k, x0, h, loss, label)
    else:   # a curved SDF: bit identities and mutant bits only (fp32 and fp64 may pick other cells near grid lines)
        want, _ = gc.guide64(k, x0[k.idx].cpu(), gc.guide_inputs(k))
        pred64, bnd = gc.clamp(k, gc.inpaint(k, want, k.idx, True)), gc.bound(k, x0[k.idx].cpu(), want, k.iters)
    if mutants:
        x0c = jc(x_t, _t(k, i), y=gc.y_dict(k, "cuda", scale=torch.ones(k.B)))
        check_mutants(k, x0, x0c, pred, pred64, bnd, label, planar)


# ------------------------------------------------------------------------------------------------ a, c
@pytest.mark.parametrize("name", list(gc.CASES))
def test_one_step(name):
    c = gc.CASES[name]
    cfg, diffusion = _model(c)
    k = gc.build(c)
    for sampler, eta, i in c["steps_run"]:
        one_step(k, cfg, diffusion, sampler, eta, i, name)
    cfg.model.engine().close()


def test_headline_steps():
    cfg = diffusion = None
    for name, c in gc.HEADLINE.items():
        if cfg is None:
            cfg, diffusion = _model(c)
        k = gc.build(c)
        for sampler, eta, i in c["steps_run"]:
            one_step(k, cfg, diffusion, sampler, eta, i, name)
    cfg.model.engine().close()


# ------------------------------------------------------------------------------------------------ b
def _chain(k, jc, diffusion, sampler, eta, xT, eps, y_fn):
    """the loop's expectation step by step: x0 = jc(x, t_i), pred = tail(hook(x0)), x = update(pred); eps[k] the
    noise of the k-th step.  Returns the samples."""
    steps = len(eps)
    x, out = xT, []
    rows = list(range(k.B))
    g = gc.guide_inputs(k, rows)
    for n, i in enumerate(range(steps - 1, -1, -1)):
        x0 = jc(x, _t(k, i), y=y_fn())
        pred, _, _ = expected(k, x0, g)
        want = _step_f32(MODE[sampler], pred.cpu().numpy(), x.cpu().numpy(), eps[n].cpu().numpy(),
                         diffusion.schedule_rows(eta)[i])
        x = torch.from_numpy(want).cuda()
        out.append(x)
    return out


@pytest.mark.parametrize("name", ["enc_joint_foot", "enc_scene_sdf_per_sample"])
def test_every_step_of_a_loop(name):
    c = gc.CASES[name]
    cfg, diffusion = _model(c)
    k = gc.build(c)
    jc = _jc(cfg, k)
    shape = (k.B, k.D, 1, k.T)
    g = torch.Generator().manual_seed(3)
    tape = torch.randn((c["steps"],) + shape, generator=g).cuda()
    xT = k.xt.cuda()
    rows = list(range(k.B))
    gi = gc.guide_inputs(k, rows)
    for sampler, eta in (("ddpm", 0.0), ("ddim", 0.0), ("ddim", 0.5)):
        kw = {} if sampler == "ddpm" else {"eta": eta}
        progf = diffusion.p_sample_loop_progressive if sampler == "ddpm" else diffusion.ddim_sample_loop_progressive
        prog = list(progf(jc, shape, noise=xT, clip_denoised=k.clip, noise_tape=tape, model_kwargs={"y": gc.y_dict(k, "cuda")},
                          **kw))
        row = diffusion.schedule_rows(eta)
        x0s = []
        for n, i in enumerate(range(c["steps"] - 1, -1, -1)):
            x_prev = xT if n == 0 else prog[n - 1]["sample"]
            x0 = jc(x_prev, _t(k, i), y=gc.y_dict(k, "cuda"))
            x0s.append(x0)
            pred, h, loss = expected(k, x0, gi)
            assert _bits_equal(pred, prog[n]["pred_xstart"]), (name, sampler, eta, i)
            check_update(MODE[sampler], row[i], pred, x_prev, tape[n], prog[n]["sample"], i)
        # the mutant: step n guided from the raw x0 of step n + 1
        for n in range(c["steps"] - 1):
            mut, _, _ = expected(k, x0s[n + 1], gi)
            assert not _bits_equal(mut, prog[n]["pred_xstart"]), (name, sampler, n)
        n = c["steps"] - 2
        pred64, bnd = check_fp64(k, x0s[n], *expected(k, x0s[n], gi)[1:], "%s %s eta %.1f step %d" % (name, sampler, eta, n))
        mut, _, _ = expected(k, x0s[n + 1], gi)
        miss = float((mut[k.idx].cpu().double().reshape(pred64.shape) - pred64).abs().max()) / bnd
        print("   mutant %-20s misses the bound %.1f-fold" % ("x0_of_next_step", miss))
        assert miss >= gc.MISS
        loops = []
        for use_graph in (True, False):
            fn = diffusion.p_sample_loop if sampler == "ddpm" else diffusion.ddim_sample_loop
            loops.append(fn(jc, shape, noise=xT, clip_denoised=k.clip, noise_tape=tape, use_graph=use_graph,
                            model_kwargs={"y": gc.y_dict(k, "cuda")}, **kw))
        print("%s %s eta %.1f: %d steps bit for bit, graph loop %s, eager loop %s"
              % (name, sampler, eta, c["steps"], _bits_equal(loops[0], prog[-1]["sample"]),
                 _bits_equal(loops[1], prog[-1]["sample"])))
        assert _bits_equal(loops[0], prog[-1]["sample"]) and _bits_equal(loops[1], prog[-1]["sample"])
        if sampler == "ddpm":
            assert _bits_equal(loops[0], prog[-1]["pred_xstart"])      # i = 0: the sample is the guided x0
    # Philox noise: the loop against the chain with the engine's own draws
    eng = cfg.model.engine()
    out = diffusion.p_sample_loop(jc, shape, clip_denoised=k.clip, noise_seed=9, model_kwargs={"y": gc.y_dict(k, "cuda")})
    xT9 = eng.philox_normal(shape, 9, 0, -1, "cuda")
    eps = [eng.philox_normal(shape, 9, 0, i, "cuda") for i in range(c["steps"] - 1, -1, -1)]
    want = _chain(k, jc, diffusion, "ddpm", 0.0, xT9, eps, lambda: gc.y_dict(k, "cuda"))[-1]
    print("%s Philox DDPM loop == chain: %s" % (name, _bits_equal(out, want)))
    assert _bits_equal(out, want)
    eng.close()


# ------------------------------------------------------------------------------------------------ d
def _loop(diffusion, m, k, xT, tape, y, use_graph=True):
    return diffusion.p_sample_loop(m, (k.B, k.D, 1, k.T), noise=xT, clip_denoised=k.clip, noise_tape=tape,
                                   use_graph=use_graph, model_kwargs={"y": y})


def test_captured_graph_follows_new_descriptors():
    c = gc.CASES["enc_scene_sdf_per_sample"]
    cfg, diffusion = _model(c)
    k = gc.build(c)
    tape = torch.randn((c["steps"], k.B, k.D, 1, k.T), generator=torch.Generator().manual_seed(4)).cuda()
    xT = k.xt.cuda()
    A = k.target.clone().cuda()
    y = lambda: gc.y_dict(k, "cuda", joint_target=A)          # noqa: E731
    first = _loop(diffusion, _jc(cfg, k), k, xT, tape, y())   # captures the step graph with lambda_1, targets A

    def check(label, jc, kk, y_fn):
        graph = _loop(diffusion, jc, kk, xT, tape, y_fn())
        eager = _loop(diffusion, jc, kk, xT, tape, y_fn(), use_graph=False)
        chain = _chain(kk, jc, diffusion, "ddpm", 0.0, xT, list(tape), y_fn)[-1]
        ok = _bits_equal(graph, eager), _bits_equal(graph, chain), not _bits_equal(graph, first)
        print("replay after %s: == eager %s, == chain %s, differs from the first loop %s" % (label, *ok))
        assert all(ok), label
    # a new lambda and K
    k2 = SimpleNamespace(**dict(vars(k), step=k.step * 0.5, iters=4))
    k2.target = A.cpu()
    check("a new lambda and K", _jc(cfg, k2, step=k2.step, iters=k2.iters), k2, y)
    # targets B in another tensor
    Bt = (k.target + 0.1 * torch.randn(k.target.shape, generator=torch.Generator().manual_seed(5))).cuda()
    kb = SimpleNamespace(**dict(vars(k), target=Bt.cpu()))
    check("targets in another tensor", _jc(cfg, kb), kb, lambda: gc.y_dict(kb, "cuda", joint_target=Bt))
    # A edited in place (the engine reads the caller's tensor)
    _loop(diffusion, _jc(cfg, k), k, xT, tape, y())
    A.add_(0.07)
    ka = SimpleNamespace(**dict(vars(k), target=A.cpu()))
    check("targets edited in place", _jc(cfg, ka), ka, y)
    # new grids
    sdf = gc._planar(k.B, [(0.2, 0.5 - 0.1 * b, 0.3) for b in range(k.B)])
    ter = gc._planar(1, [(0.1, -0.2, 0.1)])
    kg = SimpleNamespace(**dict(vars(ka), sdf=sdf, terrain=b200mdm.SceneGrid(ter.values[0], ter.origin, ter.cell)))
    check("new grids", _jc(cfg, kg), kg, lambda: gc.y_dict(kg, "cuda", joint_target=A))
    cfg.model.engine().close()


def test_feature_sequence_against_fresh_engines():
    c = gc.CASES["enc_scene_sdf_per_sample"]
    cfg, diffusion = _model(c)
    k = gc.build(c)
    tape = torch.randn((c["steps"], k.B, k.D, 1, k.T), generator=torch.Generator().manual_seed(6)).cuda()
    xT = k.xt.cuda()
    joint = dict(joint_target=k.target.cuda(), joint_weight=k.weight.cuda())
    base = dict(mask=k.inp["mask"].cuda(), lengths=k.lengths.cuda(), text_embed=k.inp["text_embed"].cuda(),
                scale=k.scale.cuda())
    foot = dict(contact_weight=gc.CW, floor_weight=gc.FW, floor_height=gc.FH)
    scene = dict(obstacle_weight=gc.OW, obstacle_margin=gc.R)
    seq = [("unguided", None, {}),
           ("joint", {}, joint),
           ("joint + foot", foot, joint),
           ("joint + foot + scene", dict(foot, **scene), dict(joint, obstacle_sdf=k.sdf, terrain=k.terrain)),
           ("joint", {}, joint),
           ("foot weights 0 + scene", dict(scene, contact_weight=0.0, floor_weight=0.0), dict(joint, obstacle_sdf=k.sdf)),
           ("unguided", None, {})]

    def run(m_cfg, kw, extra):
        m = m_cfg if kw is None else b200mdm.JointControlSampleModel(m_cfg, k.mean, k.std, k.step, k.iters, **kw)
        return _loop(diffusion, m, k, xT, tape, dict(base, **extra))
    for label, kw, extra in seq:
        got = run(cfg, kw, extra)
        fresh, _ = _model(c)
        want = run(fresh, kw, extra)
        fresh.model.engine().close()
        print("after the sequence, %-24s == a fresh engine: %s" % (label, _bits_equal(got, want)))
        assert _bits_equal(got, want), label
    cfg.model.engine().close()


def test_two_workspaces():
    ca = gc.CASES["enc_scene_sdf_per_sample"]
    cb = dict(gc.CASES["enc_joint_foot"], B=5, T=60, lengths=[60, 44, 31, 60, 12], scales=[2.5, 7.5, 1.0, 0.0, 2.5])
    cfg, diffusion = _model(ca)
    ka, kb = gc.build(ca), gc.build(cb, seed=2)
    tapes = {id(kk): torch.randn((ca["steps"], kk.B, kk.D, 1, kk.T), generator=torch.Generator().manual_seed(kk.B)).cuda()
             for kk in (ka, kb)}

    def run(m_cfg, kk):
        return _loop(diffusion, _jc(m_cfg, kk), kk, kk.xt.cuda(), tapes[id(kk)], gc.y_dict(kk, "cuda"))
    got = [run(cfg, kk) for kk in (ka, kb, ka, kb)]
    for n, kk in enumerate((ka, kb)):
        fresh, _ = _model(ca)
        want = run(fresh, kk)
        fresh.model.engine().close()
        ok = _bits_equal(got[n], want), _bits_equal(got[n + 2], want)
        print("workspace B=%d T=%d: first loop == fresh engine %s, after the other workspace %s" % (kk.B, kk.T, *ok))
        assert all(ok)
    cfg.model.engine().close()


def test_kernel_count_of_a_guided_step():
    c = gc.CASES["enc_scene_sdf_per_sample"]
    cfg, diffusion = _model(c)
    k = gc.build(c)
    eng = cfg.model.engine()
    x_t, noise = k.xt.cuda(), k.noise.cuda()
    joint = dict(joint_target=k.target.cuda(), joint_weight=k.weight.cuda())
    cases = [("unguided", cfg, {}),
             ("joint", b200mdm.JointControlSampleModel(cfg, k.mean, k.std, k.step, k.iters), joint),
             ("joint + foot", _jc(cfg, k, obstacle_weight=0.0), joint),
             ("joint + foot + scene", _jc(cfg, k), dict(joint, obstacle_sdf=k.sdf, terrain=k.terrain))]
    counts = {}
    for label, m, extra in cases:
        y = dict(mask=k.inp["mask"].cuda(), lengths=k.lengths.cuda(), text_embed=k.inp["text_embed"].cuda(),
                 scale=k.scale.cuda(), **extra)
        diffusion.p_sample(m, x_t, _t(k, 3), clip_denoised=False, model_kwargs={"y": y}, noise=noise)
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        eng.sample_step(_lib.MODE_DDPM, 3, x_t, noise)
        torch.cuda.synchronize()
        counts[label] = eng.launch_count()
    print("launches of one step: %s" % counts)
    assert counts["joint"] == counts["unguided"] + 1
    assert counts["joint + foot"] == counts["joint"] == counts["joint + foot + scene"]
    eng.close()
