"""Time joint-position control (JointControlSampleModel) at the headline shape: trans_enc, 8 layers, B = 64 motions of
196 frames, CFG 2.5, 50 DDPM steps on the engine's Philox stream and its step graph; the pelvis on every frame and both
wrists at 4 keyframes.  Unguided and guided (K = 1, 10, 50) loops run in turn on one engine (--runs rounds); each turn
starts with one untimed loop that recaptures its step graph, then times one warm loop with CUDA events.  The card's
name, power limit and SM clock are read in the same process.  Then the guidance iterations' time per launch at each K
comes from CUDA events around 5 x 20 launches of their test hook on the same shape (joint_guidance_test_kernel, which
runs the step kernel's device function and computes the loss of every iteration as well).

    python tools/time_joint_control.py [--runs 5]
"""
import argparse
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200mdm  # noqa: E402
from b200mdm.engine import joint_guidance_hook  # noqa: E402
from oracle import joint_control_oracle as jo  # noqa: E402
from time_dpm import card, spread  # noqa: E402

B, T, L, STEPS, STEP = 64, 196, 8, 50, 2e-4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_joint_control.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    mean, std = jo.motion_stats(263)
    g = torch.Generator().manual_seed(3)
    x_ref = torch.randn(B, 263, T, generator=g) * 0.5
    data = (x_ref * std[None, :, None] + mean[None, :, None]).permute(0, 2, 1)
    from oracle import ric_oracle
    target = ric_oracle.recover_from_ric(data, 22).permute(0, 2, 3, 1).contiguous()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    weight[:, 20:22, torch.arange(T // 4, T, T // 4)] = 1.0
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda(), joint_target=target.cuda(), joint_weight=weight.cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, model_kwargs={"y": y}, noise_seed=1)
    loops = {"unguided": lambda: diffusion.p_sample_loop(cfg, shape, noise=x, **kw)}
    for K in (1, 10, 50):
        jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, K)
        loops["K=%d" % K] = (lambda m: lambda: diffusion.p_sample_loop(m, shape, noise=x, **kw))(jc)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    print("library:", b200mdm._lib.LIB_PATH)
    print("card (name, power limit, SM clock, max SM clock):", card())
    t = {k: [] for k in loops}
    for _ in range(a.runs):
        for k, fn in loops.items():
            fn()                                   # recaptures this loop's step graph
            torch.cuda.synchronize()
            t[k].append(timed(fn))
    base = sorted(t["unguided"])[len(t["unguided"]) // 2]
    for k, v in t.items():
        med = sorted(v)[len(v) // 2]
        print("%-9s loop %s, per step %.3f ms, +%.3f ms per step over unguided" % (k, spread(v), med / STEPS, (med - base) / STEPS))
    x0 = torch.randn(B, 263, T, device="cuda") * 0.5
    for K in (1, 10, 50):
        args_k = (x0, mean.cuda(), std.cuda(), target.cuda(), weight.cuda(), STEP, K)
        for _ in range(3):
            joint_guidance_hook(*args_k)
        torch.cuda.synchronize()
        v = [timed(lambda: [joint_guidance_hook(*args_k) for _ in range(20)]) / 20 for _ in range(5)]
        ms = sorted(v)[len(v) // 2]
        print("guidance iterations alone (B %d, T %d), K = %2d: %s per launch over 5 x 20 launches (%.1f us per iteration)"
              % (B, T, K, spread(v), 1000 * ms / K))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
