"""Time PLMS against DDIM at BASELINE config 2's shape: trans_enc, 8 layers, B=64, 196 frames, CFG 2.5, 50 steps.
DDIM-50, PLMS-50 at order 2 and PLMS-50 at order 4 run alternately (--runs rounds), and the card's name, power limit and
SM clock are read in the same process.  A workspace keeps one captured step graph, and the three samplers' graphs differ,
so each sampler's turn starts with one untimed loop that recaptures its graph (timed separately: "first loop"); the
timed loop right after it replays a warm graph.  One line per sampler: the median and the spread of the warm loop time,
the PLMS/DDIM ratio of the medians, and the median first-loop time.  Then one loop of each sampler with plain launches
under torch.profiler: device time per kernel, summed over the loop, for the kernels whose total differs from DDIM's.

    python tools/time_plms.py [--runs 5]
"""
import argparse
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200mdm  # noqa: E402

B, T, L, STEPS = 64, 196, 8, 50


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return "%s (nvidia-smi unavailable: %s)" % (torch.cuda.get_device_name(0), exc)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_plms.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    shape = (B, 263, 1, T)
    xT = inp["tape"][0].cuda()
    kw = dict(noise=xT, clip_denoised=False, model_kwargs={"y": y})
    runs = {
        "ddim": lambda: diffusion.ddim_sample_loop(cfg, shape, noise_seed=1, **kw),
        "plms2": lambda: diffusion.plms_sample_loop(cfg, shape, order=2, **kw),
        "plms4": lambda: diffusion.plms_sample_loop(cfg, shape, order=4, **kw),
    }

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in runs.values():                      # warm-up: workspace, clocks
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    first = {k: [] for k in runs}
    for _ in range(a.runs):
        for k, fn in runs.items():
            first[k].append(timed(fn))            # recaptures this sampler's step graph
            times[k].append(timed(fn))            # warm graph
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    for k, v in times.items():
        print("%-5s B=%d T=%d L=%d %d steps CFG 2.5: median %.1f ms per loop (min %.1f, max %.1f, %d runs), %.3f x DDIM; "
              "first loop after a graph change %.1f ms"
              % (k, B, T, L, STEPS, med[k], min(v), max(v), len(v), med[k] / med["ddim"], sorted(first[k])[len(v) // 2]))
    print("card:", card())

    from torch.profiler import ProfilerActivity, profile
    per = {}
    for k in runs:
        fn = {"ddim": lambda: diffusion.ddim_sample_loop(cfg, shape, noise_seed=1, use_graph=False, **kw),
              "plms2": lambda: diffusion.plms_sample_loop(cfg, shape, order=2, use_graph=False, **kw),
              "plms4": lambda: diffusion.plms_sample_loop(cfg, shape, order=4, use_graph=False, **kw)}[k]
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        per[k] = {}
        for ev in prof.key_averages():
            if ev.device_time_total > 0:
                per[k][ev.key] = (ev.device_time_total / 1e3, ev.count)
    for k in ("plms2", "plms4"):
        tot = {n: sum(v[0] for v in per[s].values()) for n, s in (("ddim", "ddim"), (k, k))}
        print("%s: device time of all kernels %.1f ms vs DDIM %.1f ms (plain launches, one loop)" % (k, tot[k], tot["ddim"]))
        names = set(per[k]) | set(per["ddim"])
        diff = sorted(names, key=lambda n: -abs(per[k].get(n, (0, 0))[0] - per["ddim"].get(n, (0, 0))[0]))
        for n in diff[:6]:
            (tp, cp), (td, cd) = per[k].get(n, (0.0, 0)), per["ddim"].get(n, (0.0, 0))
            print("    %+8.2f ms  %s: %.2f ms / %d launches vs DDIM %.2f ms / %d" % (tp - td, n[:90], tp, cp, td, cd))


if __name__ == "__main__":
    main()
