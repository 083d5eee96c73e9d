"""TEST INFRASTRUCTURE ONLY.  Generates the fixtures of the CLIP-conditioned decoder with a timestep token
(arch='trans_dec', text_encoder_type='clip', emb_trans_dec=True) under tests/golden/ by running the UNMODIFIED
reference (via oracle/ref_harness.py) on CPU:

    python -m oracle.gen_golden_dec_emb

Files
  dec_emb_small.npz  L=2, B=3, T=24, 4 steps, lengths 24/17/5, per-sample scales 2.5/1/7.5: single forwards (cond,
                     uncond, CFG) at t=2; the DDPM loop, DDIM (eta 0) and inpainting loop outputs; a mask_frames=False
                     model (CFG forward and DDPM loop); the single target encoder (CFG forward, DDPM loop, g).
  dec_emb_c1.npz     L=8, B=1, T=196, 50 steps, CFG 2.5: the final sample.
Weights: synthetic_state_dict(arch="trans_dec", cond_dim=512); inputs: synthetic_inputs / synthetic_target_inputs
(the seeds are in each file's `meta`).
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")
OUT = os.path.join(ROOT, "tests", "golden")


def _args(**over):
    return rh.default_args(arch="trans_dec", emb_trans_dec=True, text_encoder_type="clip", **over)


def _y(inp, scale=True, **extra):
    y = dict(mask=inp["mask"], lengths=inp["lengths"], text_embed=inp["text_embed"], **extra)
    if scale:
        y["scale"] = inp["scale"]
    return y


def gen_dec_emb_small():
    ns = rh.load_reference()
    L, steps, B, T = 2, 4, 3, 24
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=9)
    inp = syn.synthetic_inputs(B, nframes=T, steps=steps, seed=15, lengths=[24, 17, 5], scale=torch.tensor([2.5, 1.0, 7.5]))
    tg = syn.synthetic_target_inputs(B, seed=5)
    shape = (B, 263, 1, T)
    out = {"meta": np.array(["trans_dec clip emb_trans_dec L=2 steps=4 B=3 T=24 weights_seed=9 inputs_seed=15 "
                             "lengths=24,17,5 scales=2.5,1,7.5 inpaint_seed=5 (first 8 frames) target=single,seed=5"])}
    x = inp["tape"][0]
    t = torch.full((B,), 2, dtype=torch.long)
    with torch.no_grad():
        model, diff = rh.build(_args(layers=L, diffusion_steps=steps), state_dict=sd)
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        out["fwd_cond"] = model(x, t, y=_y(inp, False)).numpy()
        out["fwd_uncond"] = model(x, t, y=_y(inp, False, uncond=True)).numpy()
        out["fwd_cfg"] = cfg(x, t, y=_y(inp)).numpy()
        with rh.noise_tape(inp["tape"]):
            out["ddpm"] = diff.p_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": _y(inp)}).numpy()
        with rh.noise_tape(inp["tape"]):
            out["ddim_eta0"] = diff.ddim_sample_loop(cfg, shape, clip_denoised=False, eta=0.0,
                                                     model_kwargs={"y": _y(inp)}).numpy()
        rng = np.random.default_rng(5)
        motion = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
        imask = torch.zeros(shape, dtype=torch.bool)
        imask[..., :8] = True
        with rh.noise_tape(inp["tape"]):
            out["ddpm_inpaint"] = diff.p_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={
                "y": _y(inp, inpainting_mask=imask, inpainted_motion=motion)}).numpy()
        out["inpaint_motion"] = motion.numpy()

        # the released checkpoint's args.json predates mask_frames: no key mask at all
        model, diff = rh.build(_args(layers=L, diffusion_steps=steps, mask_frames=False), state_dict=sd)
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        out["nomask_fwd_cfg"] = cfg(x, t, y=_y(inp)).numpy()
        with rh.noise_tape(inp["tape"]):
            out["nomask_ddpm"] = diff.p_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": _y(inp)}).numpy()

        sdt = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=9, target_encoder="single")
        model, diff = rh.build(_args(layers=L, diffusion_steps=steps, multi_target_cond=True, multi_encoder_type="single",
                                     target_enc_layers=1), state_dict=sdt)
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        ty = dict(target_cond=tg["target_cond"], target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
        out["target_fwd_cfg"] = cfg(x, t, y=_y(inp, **ty)).numpy()
        with rh.noise_tape(inp["tape"]):
            out["target_ddpm"] = diff.p_sample_loop(cfg, shape, clip_denoised=False, model_kwargs={"y": _y(inp, **ty)}).numpy()
        out["target_g"] = model.embed_target_cond(tg["target_cond"], tg["target_joint_names"], tg["is_heading"]).numpy()
    np.savez_compressed(os.path.join(OUT, "dec_emb_small.npz"), **out)
    print("dec_emb_small.npz:", {k: v.shape for k, v in out.items() if k != "meta"})


def gen_dec_emb_c1():
    ns = rh.load_reference()
    L, steps, B, T = 8, 50, 1, 196
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=0)
    model, diff = rh.build(_args(layers=L, diffusion_steps=steps), state_dict=sd)
    cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
    inp = syn.synthetic_inputs(B, nframes=T, steps=steps, seed=10)
    with torch.no_grad(), rh.noise_tape(inp["tape"]):
        ref = diff.p_sample_loop(cfg, (B, 263, 1, T), clip_denoised=False, model_kwargs={"y": _y(inp)})
    np.savez_compressed(os.path.join(OUT, "dec_emb_c1.npz"), sample=ref.numpy(),
                        meta=np.array(["trans_dec clip emb_trans_dec L=8 steps=50 B=1 T=196 weights_seed=0 inputs_seed=10 "
                                       "scale=2.5"]))
    print("dec_emb_c1.npz:", tuple(ref.shape), float(ref.abs().mean()))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_num_threads(8)
    gen_dec_emb_small()
    gen_dec_emb_c1()
