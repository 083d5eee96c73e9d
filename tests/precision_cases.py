"""The model kinds of tests/test_precision_margin_gpu.py (trans_enc text with CFG, a2m without it, DiP, the CLIP
decoder) at L = 8 and their real shapes, two samples each: seeded inputs, the synthetic checkpoint with stress options
(make_sd), layer 0's probe for oracle/weight_families.py, the engine's guided forward and DDIM loop (engine, needs a
GPU), and the same forward and loop in the fp32 oracle, whose `cast` may be a mdm_oracle.Sites emulation."""
import importlib
from types import SimpleNamespace

import torch

import b200mdm
from conftest import default_args
from oracle import dec_emb_oracle as deo, mdm_oracle as mo, schedule_oracle as so, weight_families as wf

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")

L, STEPS, T_HI, T_LO = 8, 10, 9, 1
SCALE = torch.tensor([2.5, 7.5])


def rel_err_per_sample(a, b):
    """||a - b||_F / ||b||_F of each batch index (dim 0)."""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).flatten(1).norm(dim=1) / b.flatten(1).norm(dim=1)


def _tables():
    return so.diffusion_tables(so.named_betas("cosine", STEPS))


def _create(args, dataset=None):
    return b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace(**(dataset or {}))))


def _load(model, sd):
    b200mdm.load_model_wo_clip(model, sd)
    return model.to("cuda").eval()


def _runners(net, diffusion, shape, y, inp):
    """(forward(x, t), loop()) of the engine: one (guided) forward at model timestep t, a DDIM loop over the tape."""
    yc = {k: (v.cuda() if torch.is_tensor(v) else tuple(u.cuda() for u in v)) for k, v in y.items()}
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()

    def forward(x, t):
        return net(x.cuda(), torch.full((shape[0],), t, dtype=torch.long, device="cuda"), y=yc).cpu()

    def loop():
        return diffusion.ddim_sample_loop(net, shape, noise=xT, clip_denoised=False, eta=0.0, model_kwargs={"y": yc},
                                          noise_tape=tape).cpu()
    return forward, loop


def _enc_text():
    B, T = 2, 196
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=STEPS, seed=71, lengths=[196, 120], scale=SCALE)
    te, ln, sc = inp["text_embed"], inp["lengths"], inp["scale"]

    def engine(sd):
        model, diffusion = _create(default_args(layers=L, diffusion_steps=STEPS))
        cfg = b200mdm.ClassifierFreeSampleModel(_load(model, sd))
        return _runners(cfg, diffusion, (B, 263, 1, T), dict(mask=inp["mask"], lengths=ln, text_embed=te, scale=sc), inp)
    return SimpleNamespace(
        sites=mo.ENC_SITES, inp=inp, engine=engine,
        make_sd=lambda **o: syn.synthetic_state_dict(num_layers=L, seed=70, **o),
        probe=wf.enc_probe(inp["tape"][0], T_HI, te, ln),
        forward=lambda W, x, t, cast: mo.cfg_denoise_enc(W, x, t, te, sc, ln, cast=cast),
        loop=lambda W, cast, tape: mo.sample_loop(W, _tables(), list(range(STEPS)), tape, te, sc, ln, sampler="ddim",
                                                  cast=cast))


def _a2m():
    B, T = 2, 60
    inp = b200mdm.synthetic_inputs(B, njoints=25, nfeats=6, nframes=T, steps=STEPS, seed=72, lengths=[60, 45])
    ln, action = inp["lengths"], torch.tensor([[3], [11]])

    def engine(sd):
        model, diffusion = _create(default_args(layers=L, diffusion_steps=STEPS, dataset="humanact12", cond_mask_prob=0.0),
                                   dict(num_actions=12))
        return _runners(_load(model, sd), diffusion, (B, 25, 6, T), dict(mask=inp["mask"], lengths=ln, action=action), inp)
    return SimpleNamespace(
        sites=mo.ENC_SITES, inp=inp, engine=engine,
        make_sd=lambda **o: syn.synthetic_state_dict(num_layers=L, seed=73, input_feats=150, cond_mode="action",
                                                     num_actions=12, **o),
        probe=wf.enc_probe(inp["tape"][0], T_HI, None, ln, action),
        forward=lambda W, x, t, cast: mo.denoise_enc(W, x, t, None, ln, action=action, cast=cast),
        loop=lambda W, cast, tape: mo.sample_loop(W, _tables(), list(range(STEPS)), tape, None, None, ln, action=action,
                                                  sampler="ddim", cast=cast))


def _dip():
    B, ctx, pred, Mt = 2, 20, 40, 16
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, ctx, seed=74)
    inp = b200mdm.synthetic_inputs(B, nframes=pred, steps=STEPS, seed=75, lengths=[40, 27], scale=SCALE)
    ln, sc = inp["lengths"], inp["scale"]

    def engine(sd):
        model, diffusion = _create(default_args(layers=L, diffusion_steps=STEPS, arch="trans_dec", text_encoder_type="bert",
                                                context_len=ctx, pred_len=pred))
        cfg = b200mdm.ClassifierFreeSampleModel(_load(model, sd))
        y = dict(mask=inp["mask"], lengths=ln, text_embed=(enc, tmask), prefix=prefix, scale=sc)
        return _runners(cfg, diffusion, (B, 263, 1, pred), y, inp)

    def forward(W, x, t, cast):
        return mo.cfg_denoise_dec(W, x, t, enc, tmask, prefix, sc, ln, cast=cast)
    return SimpleNamespace(
        sites=mo.DIP_SITES, inp=inp, engine=engine, forward=forward,
        make_sd=lambda **o: syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=768, seed=76, **o),
        probe=wf.dip_probe(inp["tape"][0], T_HI, enc, tmask, prefix, ln),
        loop=lambda W, cast, tape: deo.sample_loop(lambda x, i: forward(W, x, i, cast), _tables(), tape, sampler="ddim"))


def _dec_emb():
    B, T = 2, 196
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=STEPS, seed=77, lengths=[196, 131], scale=SCALE)
    te, ln, sc = inp["text_embed"], inp["lengths"], inp["scale"]

    def engine(sd):
        model, diffusion = _create(default_args(layers=L, diffusion_steps=STEPS, arch="trans_dec", text_encoder_type="clip",
                                                emb_trans_dec=True))
        cfg = b200mdm.ClassifierFreeSampleModel(_load(model, sd))
        return _runners(cfg, diffusion, (B, 263, 1, T), dict(mask=inp["mask"], lengths=ln, text_embed=te, scale=sc), inp)
    return SimpleNamespace(
        sites=mo.DEC_EMB_SITES, inp=inp, engine=engine,
        make_sd=lambda **o: syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=78, **o),
        probe=wf.dec_emb_probe(inp["tape"][0], T_HI, te, ln),
        forward=lambda W, x, t, cast: deo.cfg_denoise_dec_emb(W, x, t, te, sc, ln, cast=cast),
        loop=lambda W, cast, tape: deo.sample_loop(deo.denoiser(W, list(range(STEPS)), te, sc, ln, cast=cast), _tables(),
                                                   tape, sampler="ddim"))


KINDS = {"trans_enc_text": _enc_text, "a2m": _a2m, "dip": _dip, "dec_emb": _dec_emb}


def ulp_noise(x):
    """x with about one fp32 ulp of seeded random relative noise."""
    g = torch.Generator().manual_seed(1)
    return x * (1 + 2.0 ** -23 * torch.randn(x.shape, generator=g))


def fmt(e):
    return "[" + " ".join("%.2e" % v for v in e.tolist()) + "]"
