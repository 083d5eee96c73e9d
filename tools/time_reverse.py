"""Time the DDIM inversion against DDIM sampling at BASELINE config 2's shape: trans_enc, 8 layers, B=64, 196 frames,
CFG 2.5, 50 steps.  ddim_reverse_sample_loop over the whole schedule and ddim_sample_loop (the engine's Philox noise,
so both are one engine call) run alternately (--runs rounds), and the card's name, power limit and SM clock are read in
the same process.  The two loops capture different step graphs and a workspace keeps one, so each turn starts with one
loop that recaptures its graph (timed separately: "first loop"); the timed loop right after it replays a warm graph.
Then one loop of each with plain launches under torch.profiler: device time per kernel, summed over the loop, for the
kernels whose total differs most, which includes the output GEMM of each.

    python tools/time_reverse.py [--runs 5]
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
        raise SystemExit("time_reverse.py needs a GPU")
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
    x = inp["tape"][0].cuda()

    def run(k, use_graph=True):
        if k == "ddim":
            return diffusion.ddim_sample_loop(cfg, shape, noise=x, noise_seed=1, clip_denoised=False,
                                              model_kwargs={"y": y}, use_graph=use_graph)
        return diffusion.ddim_reverse_sample_loop(cfg, x, clip_denoised=False, model_kwargs={"y": y}, use_graph=use_graph)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    names = ("ddim", "reverse")
    for k in names:                               # warm-up: workspace, clocks
        for _ in range(2):
            run(k)
    torch.cuda.synchronize()
    times = {k: [] for k in names}
    first = {k: [] for k in names}
    print("card:", card())
    for _ in range(a.runs):
        for k in names:
            first[k].append(timed(k))             # recaptures this loop's step graph
            times[k].append(timed(k))             # warm graph
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    for k, v in times.items():
        print("%-7s B=%d T=%d L=%d %d steps CFG 2.5: median %.1f ms per loop (min %.1f, max %.1f, %d runs), %.3f x DDIM; "
              "first loop after a graph change %.1f ms"
              % (k, B, T, L, STEPS, med[k], min(v), max(v), len(v), med[k] / med["ddim"], sorted(first[k])[len(v) // 2]))

    from torch.profiler import ProfilerActivity, profile
    per = {}
    for k in names:
        run(k, use_graph=False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(k, use_graph=False)
            torch.cuda.synchronize()
        per[k] = {ev.key: (ev.device_time_total / 1e3, ev.count) for ev in prof.key_averages() if ev.device_time_total > 0}
    tot = {k: sum(v[0] for v in per[k].values()) for k in names}
    print("reverse: device time of all kernels %.1f ms vs DDIM %.1f ms (plain launches, one loop)" % (tot["reverse"], tot["ddim"]))
    for k in names:
        for n, (t_ms, cnt) in per[k].items():
            if "EpiOut" in n:
                print("    %-7s output GEMM %s: %.2f ms / %d launches = %.1f us per step" % (k, n[:80], t_ms, cnt, 1e3 * t_ms / cnt))
    keys = set(per["reverse"]) | set(per["ddim"])
    for n in sorted(keys, key=lambda n: -abs(per["reverse"].get(n, (0, 0))[0] - per["ddim"].get(n, (0, 0))[0]))[:6]:
        (tr, cr), (td, cd) = per["reverse"].get(n, (0.0, 0)), per["ddim"].get(n, (0.0, 0))
        print("    %+8.2f ms  %s: %.2f ms / %d launches vs DDIM %.2f ms / %d" % (tr - td, n[:90], tr, cr, td, cd))


if __name__ == "__main__":
    main()
