"""Time DiP's autoregressive chain as engine loops (the device chain) against the host chain, one sample_fn call per chunk
(reached through a non-eligible callable), alternated in one process: trans_dec, 8 layers, 40-frame chunks with a
20-frame prefix, 196 frames (5 chunks x 10 DDPM steps), guidance 7.5, Mt = 16, torch's generator reseeded per chain as
bench.py --config dip samples -- at B = 128 (the bench's shape) and B = 1.  CUDA events around whole chains after a
warm-up; the median of --reps.  The two outputs are compared bitwise.  Prints the card name and power limit.

    python tools/time_ar_chain.py [--reps N] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200mdm  # noqa: E402

CTX, PRED, MT, STEPS, NEED = 20, 40, 16, 10, 196


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ", power limit not read"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=8, cond_mask_prob=0.1, arch="trans_dec",
                           emb_trans_dec=False, text_encoder_type="bert", pos_embed_max_len=5000, mask_frames=True,
                           pred_len=PRED, context_len=CTX, diffusion_steps=STEPS, noise_schedule="cosine", sigma_small=True,
                           lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0, autoregressive_include_prefix=False)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=8, cond_dim=768, seed=23))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    res = {"card": card(), "workload": "DiP L8 d512, 5 chunks x 10 DDPM steps, CFG 7.5, Mt 16, 196 frames"}
    for B in (128, 1):
        enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, MT, CTX, seed=35)
        tmask[:] = False
        y = dict(mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"),
                 lengths=torch.full((B,), PRED, dtype=torch.int64, device="cuda"), text_embed=(enc.cuda(), tmask.cuda()),
                 prefix=prefix.cuda(), scale=torch.full((B,), 7.5, device="cuda"))
        arms = {"device": diffusion.p_sample_loop, "host": lambda *x, **k: diffusion.p_sample_loop(*x, **k)}
        samplers = {k: b200mdm.AutoRegressiveSampler(args, f, required_frames=NEED) for k, f in arms.items()}
        outs, times = {}, {k: [] for k in arms}

        def run(k):
            torch.cuda.manual_seed(35)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = samplers[k].sample(cfg, (B, 263, 1, NEED), clip_denoised=False, model_kwargs={"y": y})
            e1.record()
            torch.cuda.synchronize()
            return out, e0.elapsed_time(e1)
        for _ in range(3):
            for k in arms:
                outs[k], _ = run(k)
        for _ in range(a.reps):
            for k in arms:
                outs[k], t = run(k)
                times[k].append(t)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        res["B%d" % B] = dict(device_ms=med["device"], host_ms=med["host"], speedup=med["host"] / med["device"],
                              device_min_ms=min(times["device"]), host_min_ms=min(times["host"]),
                              bitwise_equal=bool(torch.equal(outs["device"], outs["host"])))
        print("B=%d: device chain %.3f ms, host chain %.3f ms (median of %d), host/device %.3fx, bitwise equal %s"
              % (B, med["device"], med["host"], a.reps, med["host"] / med["device"], res["B%d" % B]["bitwise_equal"]))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
