"""Time the samplers against DDIM at BASELINE config 2's shape: trans_enc, 8 layers, B=64, 196 frames, CFG 2.5, 50 steps.
DDIM (the engine's Philox noise, so one engine call per loop), PLMS at order 2 and 4, and the DDIM inversion over the
whole schedule run alternately (--runs rounds), and the card's name, power limit and SM clock are read in the same
process.  A workspace keeps one captured step graph and the samplers' graphs differ, so each sampler's turn starts with
one loop that recaptures its graph (timed apart: "first loop"); the timed loop right after it replays a warm graph.
One line per sampler: median and spread of the first and the warm loop, and the ratio of the warm medians to DDIM's.
Then one loop of each with plain launches under torch.profiler: the output GEMM's device time per step, and the kernels
whose totals differ most from DDIM's.  B200MDM_LIB selects the library, so two builds of the same ABI can be compared.

    python tools/time_samplers.py [--runs 5]
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
OUT_GEMM = "EpiOut"   # substring of every output-GEMM instantiation's kernel name


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return "%s (nvidia-smi unavailable: %s)" % (torch.cuda.get_device_name(0), exc)


def spread(v):
    s = sorted(v)
    return "%.1f ms (%.1f-%.1f)" % (s[len(s) // 2], s[0], s[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_samplers.py needs a GPU")
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
    kw = dict(clip_denoised=False, model_kwargs={"y": y})
    samplers = {
        "ddim": lambda g: diffusion.ddim_sample_loop(cfg, shape, noise=x, noise_seed=1, use_graph=g, **kw),
        "plms2": lambda g: diffusion.plms_sample_loop(cfg, shape, noise=x, order=2, use_graph=g, **kw),
        "plms4": lambda g: diffusion.plms_sample_loop(cfg, shape, noise=x, order=4, use_graph=g, **kw),
        "reverse": lambda g: diffusion.ddim_reverse_sample_loop(cfg, x, use_graph=g, **kw),
    }

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(True)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    print("library:", b200mdm._lib.LIB_PATH)
    for fn in samplers.values():                  # warm-up: workspace, clocks
        for _ in range(2):
            fn(True)
    torch.cuda.synchronize()
    warm = {k: [] for k in samplers}
    first = {k: [] for k in samplers}
    print("card:", card())
    for _ in range(a.runs):
        for k, fn in samplers.items():
            first[k].append(timed(fn))            # recaptures this sampler's step graph
            warm[k].append(timed(fn))             # warm graph
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in warm.items()}
    for k in samplers:
        print("%-7s B=%d T=%d L=%d %d steps CFG 2.5, %d runs: warm loop %s, %.3f x DDIM; first loop %s"
              % (k, B, T, L, STEPS, len(warm[k]), spread(warm[k]), med[k] / med["ddim"], spread(first[k])))

    from torch.profiler import ProfilerActivity, profile
    per = {}
    for k, fn in samplers.items():
        fn(False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(False)
            torch.cuda.synchronize()
        per[k] = {ev.key: (ev.device_time_total / 1e3, ev.count) for ev in prof.key_averages() if ev.device_time_total > 0}
    for k in samplers:
        out = [(t_ms, cnt) for n, (t_ms, cnt) in per[k].items() if OUT_GEMM in n]
        t_ms, cnt = sum(o[0] for o in out), sum(o[1] for o in out)
        print("%-7s output GEMM %.2f ms / %d launches = %.1f us per launch; device time of all kernels %.1f ms "
              "(plain launches, one loop)" % (k, t_ms, cnt, 1e3 * t_ms / max(cnt, 1), sum(v[0] for v in per[k].values())))
    for k in samplers:
        if k == "ddim":
            continue
        names = set(per[k]) | set(per["ddim"])
        for n in sorted(names, key=lambda n: -abs(per[k].get(n, (0, 0))[0] - per["ddim"].get(n, (0, 0))[0]))[:4]:
            (tk, ck), (td, cd) = per[k].get(n, (0.0, 0)), per["ddim"].get(n, (0.0, 0))
            print("    %-7s %+8.2f ms  %s: %.2f ms / %d launches vs DDIM %.2f ms / %d" % (k, tk - td, n[:90], tk, ck, td, cd))


if __name__ == "__main__":
    main()
