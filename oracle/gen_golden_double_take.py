"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/double_take_small.npz by running the UNMODIFIED reference's samplers
(diffusion/gaussian_diffusion.py, via oracle/ref_harness.py) on CPU with init_image / skip_timesteps around
oracle/double_take_oracle.SoftInpaintWrapper, which wraps the reference's own ClassifierFreeSampleModel:

    python -m oracle.gen_golden_double_take

Windows: 5 windows as motions of 3 and 2 (motion_start = [1, 0, 0, 1, 0]), lengths 24 / 20 / 24 / 16 / 24, T = 24,
CFG scales per window 2.5 / 1.0 / 7.5 / 2.5 / 4.0 (oracle/gen_golden_handshake.SMALL), h = 4, m = 3: three transitions of
Lt = 10 frames taking the scales 1.0, 7.5 and 4.0.  L = 2, 8-step cosine schedule, k = skip_timesteps = 3 (5 steps run).
  x_init                         the transitions gathered from `windows` (0.8 N(0, 1), default_rng(7))
  enc_ddpm, enc_ddim, enc_plms   p_sample_loop, ddim_sample_loop (eta 0), plms_sample_loop (order 2) of trans_enc + CLIP
                                 on the transition batch, clip_denoised=False
  enc_ddpm_clip                  p_sample_loop, clip_denoised=True
  dec_ddpm                       p_sample_loop of the CLIP decoder with a timestep token (trans_dec, emb_trans_dec)
  e2e_take1                      the reference's take 1: p_sample_loop around HandshakeWrapper (h = 4) on the windows'
                                 inputs (handshake_small's inputs and tape)
  e2e_take2                      ddim_sample_loop (eta 0) of the transitions of e2e_take1
  e2e_motion0, e2e_motion1       the stitched motions of e2e_take1 with e2e_take2 pasted in
The transition batch's noise tape is [x_T, eps...] of take2_tape(), torch.Generator seeded with TAPE_SEED.
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import double_take_oracle as dt  # noqa: E402
from oracle import gen_golden_handshake as gh  # noqa: E402
from oracle import handshake_oracle as ho  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")
OUT = os.path.join(ROOT, "tests", "golden")

SMALL = dict(gh.SMALL, steps=8, h=4, m=3, k=3, windows_seed=7)
TAPE_SEED = 17


def windows(c=SMALL):
    shape = (c["B"], 263, 1, c["T"])
    return torch.from_numpy((0.8 * np.random.default_rng(c["windows_seed"]).standard_normal(shape)).astype(np.float32))


def take2_tape(n, c=SMALL):
    """[x_T, eps_{n_run-1}, ..., eps_0] of the transition batch [n, 263, 1, Lt]."""
    Lt = 2 * c["m"] + c["h"]
    g = torch.Generator().manual_seed(TAPE_SEED)
    return list(torch.randn((c["steps"] - c["k"] + 1, n, 263, 1, Lt), generator=g).unbind(0))


def window_inputs(c=SMALL):
    """(synthetic inputs of the windows, y with the windows' scales)."""
    inp, _, y = gh.small_inputs(c)
    return inp, dict(y, scale=inp["scale"])


def _take2(diff, model, sampler, x_init, y_t, tape, clip=False):
    shape = tuple(x_init.shape)
    kw = dict(clip_denoised=clip, model_kwargs={"y": y_t}, skip_timesteps=SMALL["k"], init_image=x_init)
    if sampler == "plms":
        with rh.noise_tape(tape[:1]):
            return diff.plms_sample_loop(model, shape, order=2, **kw)
    with rh.noise_tape(tape):
        if sampler == "ddim":
            return diff.ddim_sample_loop(model, shape, eta=0.0, **kw)
        return diff.p_sample_loop(model, shape, **kw)


def gen_small():
    c = SMALL
    ns = rh.load_reference()
    inp, y = window_inputs()
    ln, ms = y["lengths"], y["motion_start"]
    W = windows()
    x_init = dt.gather(W, ln, ms, c["h"], c["m"])
    n = x_init.shape[0]
    tape = take2_tape(n)
    out = {"meta": np.array(["double take small %s" % c]), "x_init": x_init.numpy()}
    with torch.no_grad():
        args = rh.default_args(layers=c["L"], diffusion_steps=c["steps"])
        model, diff = rh.build(args, state_dict=syn.synthetic_state_dict(num_layers=c["L"], seed=c["weights_seed"]))
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        soft = dt.SoftInpaintWrapper(cfg)
        y_t = dt.transition_y(y, ln, ms, c["h"], c["m"], x_init)
        for s in ("ddpm", "ddim", "plms"):
            out["enc_" + s] = _take2(diff, soft, s, x_init, dict(y_t), tape).numpy()
        out["enc_ddpm_clip"] = _take2(diff, soft, "ddpm", x_init, dict(y_t), tape, clip=True).numpy()
        # the reference's take 1 (handshake_small's inputs), then take 2 of its transitions
        with rh.noise_tape(inp["tape"]):
            t1 = diff.p_sample_loop(ho.HandshakeWrapper(cfg, c["h"]), (c["B"], 263, 1, c["T"]), clip_denoised=False,
                                    model_kwargs={"y": dict(y)})
        xi = dt.gather(t1, ln, ms, c["h"], c["m"])
        t2 = _take2(diff, soft, "ddim", xi, dt.transition_y(y, ln, ms, c["h"], c["m"], xi), tape)
        out["e2e_take1"], out["e2e_take2"] = t1.numpy(), t2.numpy()
        for i, mo in enumerate(dt.paste(dt.stitch(t1, ln, ms, c["h"]), t2, ln, ms, c["h"], c["m"])):
            out["e2e_motion%d" % i] = mo.numpy()
        dargs = rh.default_args(layers=c["L"], diffusion_steps=c["steps"], arch="trans_dec", emb_trans_dec=True,
                                text_encoder_type="clip")
        dec, ddiff = rh.build(dargs, state_dict=syn.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=512,
                                                                         seed=c["dec_weights_seed"]))
        dsoft = dt.SoftInpaintWrapper(ns.sampler_util.ClassifierFreeSampleModel(dec))
        out["dec_ddpm"] = _take2(ddiff, dsoft, "ddpm", x_init, dict(y_t), tape).numpy()
    for k, v in out.items():
        if k != "meta":
            print(k, v.shape, float(np.abs(v).mean()))
    path = os.path.join(OUT, "double_take_small.npz")
    np.savez_compressed(path, **out)
    print("double_take_small.npz:", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_num_threads(8)
    gen_small()
