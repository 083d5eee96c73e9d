"""Time goal-directed DiP chains (AutoRegressiveSampler with y['target_world'], one waypoint per chunk) against the same
device chain with a static y['target_cond'], alternated in one process: trans_dec with the multi target encoder,
8 layers, 40-frame chunks with a 20-frame prefix, 196 frames (5 chunks x 10 DDPM steps), guidance 7.5, Mt = 16 -- at
B = 128 (bench.py --config dip's shape).  CUDA events around whole chains after a warm-up; the median of --reps.  The
difference is the cost of the 4 chunk boundaries' two launches each.  Also times b200mdm_chunk_frame alone at that
shape.  Prints the card name and power limit.

    python tools/time_goal_chain.py [--reps N] [--out FILE.json]"""
import argparse
import json
import math
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200mdm  # noqa: E402
from b200mdm.engine import Engine  # noqa: E402
from time_ar_chain import card  # noqa: E402

CTX, PRED, MT, STEPS, NEED, B = 20, 40, 16, 10, 196, 128


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=8, cond_mask_prob=0.1, arch="trans_dec",
                           emb_trans_dec=False, text_encoder_type="bert", pos_embed_max_len=5000, mask_frames=True,
                           pred_len=PRED, context_len=CTX, diffusion_steps=STEPS, noise_schedule="cosine", sigma_small=True,
                           lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0, autoregressive_include_prefix=True,
                           multi_target_cond=True, multi_encoder_type="multi", target_enc_layers=1)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=8, cond_dim=768, seed=23,
                                                                   target_encoder="multi"))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    n_chunks = -(-NEED // PRED)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, MT, CTX, seed=35)
    tmask[:] = False
    tg = b200mdm.synthetic_target_inputs(B, seed=5)
    g = torch.Generator().manual_seed(9)
    n_ext = tg["target_cond"].shape[1]
    goal = torch.randn(n_chunks, B, n_ext, 3, generator=g) * 2.0
    goal[..., -1, 0] = torch.rand(n_chunks, B, generator=g) * 2 * math.pi - math.pi
    base = dict(mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"),
                lengths=torch.full((B,), PRED, dtype=torch.int64, device="cuda"), text_embed=(enc.cuda(), tmask.cuda()),
                prefix=prefix.cuda(), scale=torch.full((B,), 7.5, device="cuda"),
                target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    ys = {"goal": dict(base, target_world=goal.cuda()), "static": dict(base, target_cond=goal[0].cuda())}
    gs = torch.Generator().manual_seed(10)
    mean, std = (torch.randn(263, generator=gs) * 0.1).cuda(), (0.5 + torch.rand(263, generator=gs)).cuda()
    s = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, required_frames=NEED, mean=mean, std=std)
    times = {k: [] for k in ys}

    def run(k):
        torch.cuda.manual_seed(35)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s.sample(cfg, (B, 263, 1, NEED), clip_denoised=False, model_kwargs={"y": ys[k]})
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    for _ in range(3):
        for k in ys:
            run(k)
    for _ in range(a.reps):
        for k in ys:
            times[k].append(run(k))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    # the boundary kernel alone, at the chain's shape: B samples, 40 frames
    carry = torch.zeros(B, 6, dtype=torch.float64, device="cuda")
    frames = torch.randn(B, 263, 1, PRED, device="cuda")
    gd = goal[0].cuda()
    for _ in range(10):
        Engine.chunk_frame(carry, frames, mean, std, gd)
    n_k = 200
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_k):
        Engine.chunk_frame(carry, frames, mean, std, gd)
    e1.record()
    torch.cuda.synchronize()
    k_us = e0.elapsed_time(e1) * 1000.0 / n_k
    res = {"card": card(), "workload": "DiP L8 d512 multi target encoder, B=128, 5 chunks x 10 DDPM steps, CFG 7.5, Mt 16, "
           "196 frames + 20-frame prefix", "goal_ms": med["goal"], "static_ms": med["static"],
           "goal_min_ms": min(times["goal"]), "static_min_ms": min(times["static"]),
           "per_boundary_us": (med["goal"] - med["static"]) * 1000.0 / (n_chunks - 1),
           "chunk_frame_call_us": k_us, "reps": a.reps}
    print("B=%d: goal chain %.3f ms, static-target chain %.3f ms (median of %d); %.1f us per boundary; "
          "chunk_frame call alone %.1f us (host-timed enqueue included)"
          % (B, med["goal"], med["static"], a.reps, res["per_boundary_us"], k_us))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
