"""GPU: DDIM inversion (ddim_reverse_sample / ddim_reverse_sample_loop / ddim_reverse_sample_loop_progressive).

  * the reverse epilogue bit for bit against a torch fp32 restatement of the reference's update, fed with the engine's
    own pred_xstart, at i = 0, a middle index and n - 1, with and without the clamp and inpainting; three mutants of
    the restatement (sqrt(abp) for sqrt(abn), eps from row i + 1, an fp64 combine rounded once) must differ;
  * the loop bit for bit equal to the chain of single steps and to the progressive form, with and without graph
    replay, and split into two range calls;
  * every case of tests/golden/reverse_small.npz: the last step against the reference's own sample, every step against
    the fp32 oracle, and the c2 shape at 50 steps against the fp32 oracle, all within 1e-3;
  * a reverse loop between two DDIM loops, or between two PLMS loops, changes neither; a reverse step launches what a
    DDIM step launches; a reverse call after a schedule change without its reverse table fails."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import gen_golden_reverse as gr
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import reverse_oracle as ro
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
RTOL = 1e-3


def _enc(layers, steps, seed):
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(layers=layers, diffusion_steps=steps),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=layers, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion, sd


def _y(inp, scale=True):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda())
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _small():
    c = gr.ENC
    cfg, model, diffusion, _ = _enc(c["L"], c["steps"], c["weights_seed"])
    inp, shape, imask, motion = gr.enc_inputs()
    return cfg, model, diffusion, inp, shape, imask, motion


def _t(i, b):
    return torch.full((b,), i, dtype=torch.long, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
def _update(diffusion, x, i, x0, eps_row=None, next_cols=None, f64=False):
    """ddim_reverse_sample's update (gaussian_diffusion.py:861-872), torch fp32 on the CPU, from the fp32 table values."""
    rows = torch.from_numpy(diffusion.schedule_rows(0.0))
    e = rows[i if eps_row is None else eps_row]
    sa, sb = next_cols if next_cols is not None else torch.from_numpy(diffusion.schedule_next_rows())[i]
    if f64:
        x, x0, e, sa, sb = x.double(), x0.double(), e.double(), sa.double(), sb.double()
    eps = (e[3] * x - x0) / e[4]
    return (x0 * sa + sb * eps).float()


@pytest.mark.parametrize("i", [0, 3, 5])
def test_update_bit_exact(i):
    cfg, _, diffusion, inp, shape, imask, motion = _small()
    x = inp["tape"][0].cuda()
    xc = x.cpu()
    rows = diffusion.schedule_rows(0.0)
    for clip, inpaint in ((False, False), (True, False), (False, True), (True, True)):
        y = _y(inp)
        if inpaint:
            y.update(inpainting_mask=imask.cuda(), inpainted_motion=motion.cuda())
        out = diffusion.ddim_reverse_sample(cfg, x, _t(i, shape[0]), clip_denoised=clip, model_kwargs={"y": y})
        x0, got = out["pred_xstart"].cpu(), out["sample"].cpu()
        if inpaint:
            want = motion.clamp(-1, 1) if clip else motion
            assert torch.equal(x0[imask], want[imask])
        if clip:
            assert x0.abs().max() <= 1
        assert torch.equal(got, _update(diffusion, xc, i, x0)), (i, clip, inpaint)
        if i == diffusion.num_timesteps - 1:                            # abn = 0: the sample is eps
            assert torch.equal(got, (torch.tensor(rows[i, 3]) * xc - x0) / torch.tensor(rows[i, 4]))
        abp = (torch.tensor(rows[i, 5]), torch.tensor(rows[i, 6]))     # mutant: sqrt(abp), sqrt(1 - abp)
        assert not torch.equal(got, _update(diffusion, xc, i, x0, next_cols=abp))
        if i + 1 < diffusion.num_timesteps:                             # mutant: eps from row i + 1
            assert not torch.equal(got, _update(diffusion, xc, i, x0, eps_row=i + 1))
        assert not torch.equal(got, _update(diffusion, xc, i, x0, f64=True))   # mutant: fp64 combine, rounded once


def test_loop_equals_steps():
    cfg, _, diffusion, inp, shape, _, _ = _small()
    y = _y(inp)
    x = inp["tape"][0].cuda()
    n = diffusion.num_timesteps
    chain, z = [], x
    for i in range(n):
        z = diffusion.ddim_reverse_sample(cfg, z, _t(i, shape[0]), clip_denoised=False, model_kwargs={"y": y})["sample"]
        chain.append(z)
    prog = [o["sample"] for o in diffusion.ddim_reverse_sample_loop_progressive(cfg, x, clip_denoised=False,
                                                                                model_kwargs={"y": y})]
    assert len(prog) == n and all(torch.equal(a, b) for a, b in zip(prog, chain))
    eng = cfg.model.engine()
    for use_graph in (True, False):
        loop = diffusion.ddim_reverse_sample_loop(cfg, x, clip_denoised=False, model_kwargs={"y": y}, use_graph=use_graph)
        assert torch.equal(loop, chain[-1]), use_graph
        part = diffusion.ddim_reverse_sample_loop(cfg, chain[0], clip_denoised=False, model_kwargs={"y": y},
                                                  first_index=1, n_steps=3, use_graph=use_graph)
        assert torch.equal(part, chain[3]), use_graph
        out = torch.empty_like(x)
        eng.ddim_reverse_loop_range(0, 2, x, None, 0, use_graph)
        eng.ddim_reverse_loop_range(2, n - 2, None, out, 0, use_graph)
        torch.cuda.synchronize()
        assert torch.equal(out, chain[-1]), use_graph
    assert torch.equal(x, inp["tape"][0].cuda())             # the caller's x is not clobbered by the in-place loop


# ---------------------------------------------------------------------------------------------------------------------
# Every case is held to RTOL at every step (see DESIGN.md section 2): the last step against the reference's own sample
# (the fixture), every step against the fp32 oracle, which tests/test_reverse_cpu.py pins to that sample.
def _steps(diffusion, m, x, y, clip):
    prog = [o["sample"] for o in diffusion.ddim_reverse_sample_loop_progressive(m, x, clip_denoised=clip,
                                                                                model_kwargs={"y": y})]
    loop = diffusion.ddim_reverse_sample_loop(m, x, clip_denoised=clip, model_kwargs={"y": y})
    assert torch.equal(loop, prog[-1])
    return prog


def _check(name, steps, g, denoise, tables, x, clip=False, inpaint=None):
    ref = []
    ro.reverse_loop(denoise, tables, x, clip_denoised=clip, inpaint=inpaint, collect=ref)
    assert len(steps) == len(ref)
    errs = [rel_err(s, r) for s, (r, _) in zip(steps, ref)]
    final = rel_err(steps[-1], g["%s_sample" % name])
    print("%s: relative error per step vs the fp32 oracle %s; last step vs the reference %.2e"
          % (name, " ".join("%.2e" % e for e in errs), final))
    assert max(errs) < RTOL and final < RTOL, (name, errs, final)


def test_golden_enc(golden):
    g = golden("reverse_small.npz")
    c = gr.ENC
    cfg, _, diffusion, inp, shape, imask, motion = _small()
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]), c["L"])
    f = po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], inp["lengths"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    x = inp["tape"][0]
    _check("enc", _steps(diffusion, cfg, x.cuda(), _y(inp), False), g, f, tabs, x)
    y = dict(_y(inp), inpainting_mask=imask.cuda(), inpainted_motion=motion.cuda())
    _check("enc_clip_inpaint", _steps(diffusion, cfg, x.cuda(), y, True), g, f, tabs, x, True, (imask, motion))


def test_golden_dip(golden):
    c = gr.DIP
    args = default_args(layers=c["L"], diffusion_steps=c["steps"], arch="trans_dec", text_encoder_type="bert",
                        context_len=c["ctx"], pred_len=c["pred"])
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768, seed=c["weights_seed"])
    b200mdm.load_model_wo_clip(model, sd)
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp, enc, tmask, prefix = gr.dip_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             scale=inp["scale"].cuda(), prefix=prefix.cuda())
    f = po.dec_denoiser(mo.OracleWeights(sd, c["L"]), list(range(c["steps"])), enc, tmask, prefix, inp["scale"],
                        inp["lengths"])
    x = inp["tape"][0]
    _check("dip", _steps(diffusion, cfg, x.cuda(), y, False), golden("reverse_small.npz"), f,
           so.diffusion_tables(so.named_betas("cosine", c["steps"])), x)


def test_golden_respaced(golden):
    c = gr.RESP
    _, model, _, sd = _enc(c["L"], c["base_steps"], c["weights_seed"])
    diffusion = gr.respaced_diffusion(gd, rs)
    assert diffusion.timestep_map != list(range(diffusion.num_timesteps))
    inp = gr.resp_inputs()
    f = po.enc_denoiser(mo.OracleWeights(sd, c["L"]), diffusion.timestep_map, inp["text_embed"], None, inp["lengths"])
    betas, _, _ = so.respaced(so.named_betas("cosine", c["base_steps"]), so.space_timesteps(c["base_steps"], c["respacing"]))
    x = inp["tape"][0]
    _check("respaced", _steps(diffusion, model, x.cuda(), _y(inp, scale=False), False), golden("reverse_small.npz"), f,
           so.diffusion_tables(betas), x)


def test_c2_shape_50_steps_vs_oracle():
    B, T, steps = 64, 196, 50
    cfg, _, diffusion, sd = _enc(8, steps, 0)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    out = diffusion.ddim_reverse_sample_loop(cfg, inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": _y(inp)})
    assert torch.isfinite(out).all()
    idx = [0, 31, 63]
    W = mo.OracleWeights(sd, 8)
    f = po.enc_denoiser(W, list(range(steps)), inp["text_embed"][:, idx], inp["scale"][idx], inp["lengths"][idx])
    ref = ro.reverse_loop(f, so.diffusion_tables(so.named_betas("cosine", steps)), inp["tape"][0][idx])
    err = rel_err(out[idx], ref)
    print("DDIM inversion, B=64 x 50 steps x CFG 2.5: Frobenius-relative %.3e" % err)
    assert err < RTOL


# ---------------------------------------------------------------------------------------------------------------------
def test_no_interference_and_launches():
    cfg, _, diffusion, inp, shape, _, _ = _small()
    y = _y(inp)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, model_kwargs={"y": y})
    ddim = [diffusion.ddim_sample_loop(cfg, shape, noise=x, noise_seed=5, **kw)]
    diffusion.ddim_reverse_sample_loop(cfg, x, **kw)
    ddim.append(diffusion.ddim_sample_loop(cfg, shape, noise=x, noise_seed=5, **kw))
    assert torch.equal(ddim[0], ddim[1])
    plms = [diffusion.plms_sample_loop(cfg, shape, noise=x, order=2, **kw)]
    diffusion.ddim_reverse_sample_loop(cfg, x, **kw)
    plms.append(diffusion.plms_sample_loop(cfg, shape, noise=x, order=2, **kw))
    assert torch.equal(plms[0], plms[1])
    # a reverse step launches what a DDIM step with a noise tape launches
    eng = cfg.model.engine()
    n = diffusion.num_timesteps
    for use_graph in (True, False):
        eng.ddim_reverse_loop_range(0, 1, x, None, 0, use_graph)
        eng.launch_count(reset=True)
        eng.ddim_reverse_loop_range(1, n - 1, None, None, 0, use_graph)
        rev = eng.launch_count(reset=True)
        tape = torch.zeros((n - 1,) + tuple(shape), device="cuda")
        eng.sample_loop_range(_lib.MODE_DDIM, n - 2, n - 1, x, None, tape, 0, use_graph)
        ddim_n = eng.launch_count(reset=True)
        assert rev == ddim_n, (use_graph, rev, ddim_n)
        torch.cuda.synchronize()
    # a new schedule makes the reverse table stale until it is set again
    eng.set_schedule(diffusion.schedule_rows(0.0), list(range(n)))
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.ddim_reverse_loop_range(0, n, x, None, 0, True)
    assert exc.value.code == _lib.ESTATE
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.sample_step(_lib.MODE_DDIM_REVERSE, 0, x, None, 0)
    assert exc.value.code == _lib.ESTATE
    with pytest.raises(_lib.B200MDMError) as exc:
        eng.set_schedule_next(np.zeros((n + 1, 2), dtype=np.float32))
    assert exc.value.code == _lib.EINVAL
    again = diffusion.ddim_reverse_sample_loop(cfg, x, **kw)             # _prepare sets both tables again
    assert torch.equal(again, diffusion.ddim_reverse_sample_loop(cfg, x, use_graph=False, **kw))
