"""Time the CLIP-conditioned decoder with a timestep token (trans_dec, emb_trans_dec=True) against the encoder at
BASELINE config 2's shape: 8 layers, B=64, 196 frames, CFG 2.5, 50 DDIM steps with the engine's Philox noise (one
engine call per loop).  The two models run alternately (--runs rounds) on their own engines, so each replays a warm
step graph; CUDA events time each loop.  The card's name, power limit and SM clock are read in the same process.
Then one loop of each with plain launches under torch.profiler: device time per launch of the decoder's two own
kernels (the per-step cross-attention rows and the row-bias LayerNorm, with the LayerNorm's achieved bandwidth against
the H100 SXM's 3.35 TB/s data-sheet figure) and the kernels whose totals differ most between the two models.

    python tools/time_dec_emb.py [--runs 5]
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
HBM_BYTES_PER_S = 3.35e12
KERNELS = {"cross rows": "cross_rows_kernel", "row-bias LayerNorm": "row_bias_ln_kernel"}


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


def build(arch):
    dec = arch == "decoder"
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_dec" if dec else "trans_enc", emb_trans_dec=dec, text_encoder_type="clip",
                           pos_embed_max_len=5000, mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS,
                           noise_schedule="cosine", sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec" if dec else "trans_enc", num_layers=L, seed=0)
    b200mdm.load_model_wo_clip(model, sd)
    return b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval()), diffusion


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_dec_emb.py needs a GPU")
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    loops = {}
    for arch in ("decoder", "encoder"):
        cfg, diffusion = build(arch)
        loops[arch] = (lambda c, d: lambda g: d.ddim_sample_loop(c, shape, noise=x, noise_seed=1, use_graph=g, clip_denoised=False,
                                                                 model_kwargs={"y": y}))(cfg, diffusion)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(True)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    print("library:", b200mdm._lib.LIB_PATH)
    for fn in loops.values():                      # warm-up: workspaces, graphs, clocks
        for _ in range(2):
            fn(True)
    torch.cuda.synchronize()
    print("card (before):", card())
    ms = {k: [] for k in loops}
    for _ in range(a.runs):
        for k, fn in loops.items():
            ms[k].append(timed(fn))
    print("card (after):", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    for k in loops:
        print("%-7s B=%d T=%d L=%d %d DDIM steps CFG 2.5, %d runs: warm loop %s, %.1f motions/s, %.3f x encoder"
              % (k, B, T, L, STEPS, len(ms[k]), spread(ms[k]), B / med[k] * 1e3, med[k] / med["encoder"]))

    from torch.profiler import ProfilerActivity, profile
    per = {}
    for k, fn in loops.items():
        fn(False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(False)
            torch.cuda.synchronize()
        per[k] = {ev.key: (ev.device_time_total, ev.count) for ev in prof.key_averages() if ev.device_time_total > 0}
    M = 2 * B * (T + 1)
    for label, name in KERNELS.items():
        hits = [(us, n) for key, (us, n) in per["decoder"].items() if name in key]
        us, n = sum(h[0] for h in hits), sum(h[1] for h in hits)
        line = "decoder %s: %.1f us per launch (%d launches, plain launches, one loop)" % (label, us / max(n, 1), n)
        if name == "row_bias_ln_kernel" and n:
            bytes_ = M * 2 * 1024 * 2 + 2 * B * 512 * 4      # [hi | lo] rows read and written, c rows read
            bw = bytes_ / (us / n * 1e-6)
            line += "; %d rows, %.1f MB moved: %.2f TB/s = %.0f %% of 3.35 TB/s" % (M, bytes_ / 1e6, bw / 1e12, 100 * bw / HBM_BYTES_PER_S)
        print(line)
    for k in loops:
        print("%-7s device time of all kernels %.1f ms (plain launches, one loop)" % (k, sum(v[0] for v in per[k].values()) / 1e3))
    names = set(per["decoder"]) | set(per["encoder"])
    for n in sorted(names, key=lambda n: -abs(per["decoder"].get(n, (0, 0))[0] - per["encoder"].get(n, (0, 0))[0]))[:6]:
        (td, cd), (te, ce) = per["decoder"].get(n, (0.0, 0)), per["encoder"].get(n, (0.0, 0))
        print("    decoder %+8.2f ms  %s: %.2f ms / %d launches vs encoder %.2f ms / %d" % ((td - te) / 1e3, n[:90], td / 1e3, cd,
                                                                                          te / 1e3, ce))


if __name__ == "__main__":
    main()
