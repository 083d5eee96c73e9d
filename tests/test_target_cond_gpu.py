"""GPU: target-location conditioning (multi_target_cond) through the engine -- against the reference's golden outputs,
the fp32 oracle (oracle/target_oracle.py), the plain model, and, for the device target encoder alone, an fp64
evaluation with a per-element error bound derived from the fp32 arithmetic."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from conftest import default_args, rel_err
from oracle import mdm_oracle as mo
from oracle import schedule_oracle as so
from oracle import target_oracle as to

pytestmark = pytest.mark.gpu
RTOL = 1e-3
JOINTS = b200mdm.synthetic.HML_TARGET_JOINTS


def _build(arch, encoder, L, steps, seed, layers=1):
    over = dict(layers=L, diffusion_steps=steps)
    if encoder is not None:
        over.update(multi_target_cond=True, multi_encoder_type=encoder, target_enc_layers=layers)
    if arch == "trans_dec":
        over.update(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch=arch, num_layers=L, cond_dim=768 if arch == "trans_dec" else 512, seed=seed,
                                      target_encoder=encoder, target_enc_layers=layers)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion, sd


def _target_y(tg):
    return dict(target_cond=tg["target_cond"].cuda(), target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])


def _dip_inputs(B=3, seed=13, lengths=(40, 33, 12), scale=(7.5, 2.0, 1.0), steps=3, Mt=7, dip_seed=3):
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, 20, seed=dip_seed)
    inp = b200mdm.synthetic_inputs(B, nframes=40, steps=steps, seed=seed, lengths=list(lengths), scale=torch.tensor(scale))
    return enc, tmask, prefix, inp


def _dip_y(inp, enc, tmask, prefix, scale=True):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()), prefix=prefix.cuda())
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _enc_inputs():
    return b200mdm.synthetic_inputs(4, nframes=24, steps=3, seed=14, lengths=[24, 20, 11, 6],
                                    scale=torch.tensor([2.5, 1.0, 5.0, 2.5]))


def _enc_y(inp, scale=True):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda())
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _tape(inp):
    return torch.stack(inp["tape"][1:]).cuda(), inp["tape"][0].cuda()


def _loops(diffusion, cfg, shape, y, inp):
    tape, xT = _tape(inp)
    outs = [diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape,
                                    use_graph=g) for g in (False, True)]
    assert torch.equal(outs[0], outs[1])
    return outs[0]


def test_dip_single_encoder_vs_reference_golden(golden):
    g = golden("dip_target_small.npz")
    cfg, model, diffusion, _ = _build("trans_dec", "single", 2, 3, 4)
    enc, tmask, prefix, inp = _dip_inputs()
    tg = b200mdm.synthetic_target_inputs(3, seed=5)
    x = inp["tape"][0].cuda()
    t = torch.full((3,), 1, dtype=torch.long, device="cuda")
    y = dict(_dip_y(inp, enc, tmask, prefix), **_target_y(tg))
    assert rel_err(cfg(x, t, y=y), g["fwd_cfg"]) < RTOL
    assert rel_err(cfg(x, t, y=dict(y, target_uncond=True)), g["fwd_cfg_target_uncond"]) < RTOL
    assert rel_err(_loops(diffusion, cfg, (3, 263, 1, 40), y, inp), g["ddpm"]) < RTOL


def test_enc_multi_encoder_vs_reference_golden(golden):
    g = golden("enc_target_small.npz")
    cfg, model, diffusion, _ = _build("trans_enc", "multi", 2, 3, 6)
    inp = _enc_inputs()
    tg = b200mdm.synthetic_target_inputs(4, seed=8)
    x = inp["tape"][0].cuda()
    t = torch.full((4,), 2, dtype=torch.long, device="cuda")
    assert rel_err(model(x, t, y=dict(_enc_y(inp, False), **_target_y(tg))), g["fwd_cond"]) < RTOL
    y = dict(_enc_y(inp), **_target_y(tg))
    assert rel_err(cfg(x, t, y=y), g["fwd_cfg"]) < RTOL
    assert rel_err(_loops(diffusion, cfg, (4, 263, 1, 24), y, inp), g["ddpm"]) < RTOL


def test_split_encoder_vs_oracle():
    cfg, model, _, sd = _build("trans_enc", "split", 3, 3, 9, layers=2)
    W = mo.OracleWeights(sd, 3)
    inp = b200mdm.synthetic_inputs(5, nframes=30, steps=3, seed=41, lengths=[30, 30, 17, 9, 2],
                                   scale=torch.tensor([2.5, 7.5, 1.0, 0.0, 2.5]))
    tg = b200mdm.synthetic_target_inputs(5, seed=42)
    gt = to.target_embedding(W, "split", tg["target_cond"], to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"]),
                             layers=2)
    x = inp["tape"][0]
    t = torch.full((5,), 1, dtype=torch.long)
    want = to.cfg(to.denoise_enc, inp["scale"], W, x, 1, inp["text_embed"], gt, inp["lengths"])
    assert rel_err(cfg(x.cuda(), t.cuda(), y=dict(_enc_y(inp), **_target_y(tg))), want) < RTOL
    want = to.denoise_enc(W, x, 1, inp["text_embed"], gt, inp["lengths"])
    assert rel_err(model(x.cuda(), t.cuda(), y=dict(_enc_y(inp, False), **_target_y(tg))), want) < RTOL


@pytest.mark.parametrize("arch", ["trans_enc", "trans_dec"])
def test_without_target_equals_plain_model(arch):
    """A target-conditioned model sampled without y['target_cond'] (or with target_uncond) is the plain model."""
    encoder = "single" if arch == "trans_dec" else "multi"
    cfg_t, _, diffusion, _ = _build(arch, encoder, 2, 3, 17)
    cfg_p, _, _, _ = _build(arch, None, 2, 3, 17)
    if arch == "trans_dec":
        enc, tmask, prefix, inp = _dip_inputs()
        y, shape = _dip_y(inp, enc, tmask, prefix), (3, 263, 1, 40)
        B = 3
    else:
        inp = _enc_inputs()
        y, shape = _enc_y(inp), (4, 263, 1, 24)
        B = 4
    plain = _loops(diffusion, cfg_p, shape, y, inp)
    tg = _target_y(b200mdm.synthetic_target_inputs(B, seed=3))
    with_target = _loops(diffusion, cfg_t, shape, dict(y, **tg), inp)
    assert not torch.equal(with_target, plain)
    assert torch.equal(_loops(diffusion, cfg_t, shape, y, inp), plain)             # set_cond clears the previous target
    assert torch.equal(_loops(diffusion, cfg_t, shape, dict(y, target_uncond=True, **tg), inp), plain)


def test_launches_per_step_unchanged_by_target():
    enc, tmask, prefix, inp = _dip_inputs(steps=5)
    tg = _target_y(b200mdm.synthetic_target_inputs(3, seed=3))
    y = _dip_y(inp, enc, tmask, prefix)
    tape, xT = _tape(inp)
    per_loop = {}
    for steps in (3, 5):
        cfg, model, diffusion, _ = _build("trans_dec", "single", 2, steps, 4)
        eng = model.engine()
        for name, yy in (("plain", y), ("target", dict(y, **tg))):
            for use_graph in (True, False):
                eng.launch_count(reset=True)
                diffusion.p_sample_loop(cfg, (3, 263, 1, 40), noise=xT, clip_denoised=False, model_kwargs={"y": yy},
                                        noise_tape=tape[:steps], use_graph=use_graph)
                torch.cuda.synchronize()
                per_loop[(steps, name, use_graph)] = eng.launch_count()
    for use_graph in (True, False):
        for steps in (3, 5):   # the target adds its one encoder launch per loop, and nothing per step
            assert per_loop[(steps, "target", use_graph)] == per_loop[(steps, "plain", use_graph)] + 1
        assert (per_loop[(5, "target", use_graph)] - per_loop[(3, "target", use_graph)] ==
                per_loop[(5, "plain", use_graph)] - per_loop[(3, "plain", use_graph)])


def test_dip_full_depth_target_philox_vs_oracle():
    """DiP at its released depth (8 layers) with the single target encoder and the engine's Philox noise stream."""
    B, steps, seed = 4, 5, 1234
    cfg, model, diffusion, sd = _build("trans_dec", "single", 8, steps, 27)
    W = mo.OracleWeights(sd, 8)
    enc, tmask, prefix, inp = _dip_inputs(B=B, seed=51, lengths=(40, 25, 40, 3), scale=(7.5, 2.5, 1.0, 7.5), steps=steps,
                                          Mt=11, dip_seed=52)
    tg = b200mdm.synthetic_target_inputs(B, seed=53)
    y = dict(_dip_y(inp, enc, tmask, prefix), **_target_y(tg))
    shape = (B, 263, 1, 40)
    out = diffusion.p_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": y}, noise_seed=seed)
    eng = model.engine()
    tape = [eng.philox_normal(shape, seed, 0, -1, "cuda").cpu()]
    tape += [eng.philox_normal(shape, seed, 0, i, "cuda").cpu() for i in range(steps - 1, -1, -1)]
    gt = to.target_embedding(W, "single", tg["target_cond"], to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"]))
    want = to.sample_loop_dec(W, so.diffusion_tables(so.named_betas("cosine", steps)), list(range(steps)), tape, enc, tmask,
                              prefix, gt, inp["scale"], inp["lengths"])
    assert rel_err(out, want) < RTOL


# ---------------------------------------------------------------------------------------------------------------------
# The device target encoder (target_embed_kernel) against fp64.  The bound follows the fp32 arithmetic of the kernel:
#   Linear (K products accumulated by fmaf, then + bias): |err| <= gamma_{K+1} (|W| (|x| + dx) + |b|) + |W| dx
#   SiLU h / (1 + expf(-h)) on a perturbed h: |err| <= 1.1 dh + 8 u (|s| + 1.1 dh)   (|silu'| <= 1.1; expf 2 ulp, +, /)
#   WeightedSum: sum(w) to gamma_n sum|w|, w_i / sum(w) to one more rounding, then n fmaf into the accumulator.
U = 2.0 ** -24


def _gamma(k):
    return k * U / (1 - k * U)


def _lin(w, b, x, dx):
    y = x @ w.T + b
    return y, _gamma(w.shape[1] + 1) * ((np.abs(x) + dx) @ np.abs(w).T + np.abs(b)) + dx @ np.abs(w).T


def _silu(h, dh, on=True):
    if not on:
        return h, dh
    s = h / (1 + np.exp(-h))
    return s, 1.1 * dh + 8 * U * (np.abs(s) + 1.1 * dh)


def _mlp(sd, prefix, x, n_hidden, silu=True):
    h, dh = _lin(sd[prefix + "0.weight"], sd[prefix + "0.bias"], x, np.zeros_like(x))
    for k in range(1, n_hidden + 1):
        s, ds = _silu(h, dh, silu)
        h, dh = _lin(sd[prefix + "%d.weight" % (2 * k)], sd[prefix + "%d.bias" % (2 * k)], s, ds)
    return h, dh


def _encoder64(sd, encoder, layers, target, valid, silu=True, normalise=True):
    """(g, bound) in fp64 for target [B, n, 3], valid [B, n] (float)."""
    B, n, _ = target.shape
    x = np.concatenate([target, valid[..., None]], axis=-1)
    if encoder == "single":
        return _mlp(sd, "embed_target_cond.mlp.", x.reshape(B, 4 * n), layers, silu)
    if encoder == "split":
        parts = [_mlp(sd, "embed_target_cond.mini_mlps.%d." % i, x[:, i], layers, silu) for i in range(n)]
        return np.concatenate([p[0] for p in parts], -1), np.concatenate([p[1] for p in parts], -1)
    w = sd["embed_target_cond.target_all_loc_emb.weights"]
    wt, dwt = w.sum(), _gamma(n) * np.abs(w).sum()
    nw = w / wt if normalise else w
    dnw = np.abs(nw) * (dwt / abs(wt) + U) * 1.01
    d = sd["embed_target_cond.target_loc_emb.%s.0.bias" % JOINTS[0]].shape[0]
    g, bound = np.zeros((B, d)), np.zeros((B, d))
    for b in range(B):
        acc_abs = np.zeros(d)
        for i in range(n):
            if valid[b, i] == 0:
                continue
            r, dr = _mlp(sd, "embed_target_cond.target_loc_emb.%s." % JOINTS[i], target[b, i][None], 1, silu)
            r, dr = r[0], dr[0]
            g[b] += nw[i] * r
            bound[b] += abs(nw[i]) * dr + dnw[i] * np.abs(r)
            acc_abs += (abs(nw[i]) + dnw[i]) * (np.abs(r) + dr)
        bound[b] += _gamma(n) * acc_abs
    return g, bound


@pytest.mark.parametrize("encoder,layers", [("single", 2), ("split", 1), ("multi", 1)])
def test_target_encoder_kernel_vs_fp64(encoder, layers):
    _, model, _, sd = _build("trans_enc", encoder, 1, 3, 31, layers=layers)
    sd64 = {k: v.double().numpy() for k, v in sd.items() if k.startswith("embed_target_cond.")}
    B, n = 24, len(JOINTS)
    rng = np.random.default_rng(7)
    target = (rng.standard_normal((B, n, 3)) * 2.0).astype(np.float32)
    valid = (rng.random((B, n)) < 0.5).astype(np.uint8)
    valid[::2, JOINTS.index("heading")] = 1
    valid[0] = 0                                   # no joint at all
    valid[1] = 1                                   # every joint, heading included
    got = model.engine().test_target(torch.from_numpy(target).cuda(), valid).double().cpu().numpy()
    want, bound = _encoder64(sd64, encoder, layers, target.astype(np.float64), valid.astype(np.float64))
    bound = bound + 1e-300
    ratio = np.abs(got - want) / bound
    assert ratio.max() <= 1.0, ratio.max()
    if encoder == "multi":
        assert not got[0].any()
    no_heading = valid.copy()
    no_heading[:, JOINTS.index("heading")] = 0
    mutants = {"heading dropped": _encoder64(sd64, encoder, layers, target.astype(np.float64), no_heading.astype(np.float64))[0],
               "SiLU removed": _encoder64(sd64, encoder, layers, target.astype(np.float64), valid.astype(np.float64), silu=False)[0]}
    if encoder == "multi":
        mutants["WeightedSum unnormalised"] = _encoder64(sd64, encoder, layers, target.astype(np.float64),
                                                         valid.astype(np.float64), normalise=False)[0]
    for name, m in mutants.items():
        assert (np.abs(m - want) / bound).max() >= 8.0, name
    print("%s: kernel error / bound %.3g; mutants: %s" % (encoder, ratio.max(), ", ".join(
        "%s %.3g" % (k, (np.abs(m - want) / bound).max()) for k, m in mutants.items())))
