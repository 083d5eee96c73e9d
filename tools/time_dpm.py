"""Time DPM-Solver++ (orders 1 and 2) against DDIM at BASELINE config 2's shape: trans_enc, 8 layers, B=64, 196 frames,
CFG 2.5, 20 steps respaced from a 1000-step cosine schedule.  The three samplers run alternately on the same engine
(--runs rounds); each turn starts with one loop that recaptures its step graph (untimed), then times one warm replay
with CUDA events.  The card's name, power limit and SM clock are read in the same process.  Then one loop of each with
plain launches under torch.profiler gives the output GEMM's device time per launch.

    python tools/time_dpm.py [--runs 7]
"""
import argparse
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200mdm  # noqa: E402
from b200mdm.diffusion import gaussian_diffusion as gd  # noqa: E402

B, T, L, BASE, STEPS = 64, 196, 8, 1000, "20"
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
    return "%.2f ms (%.2f-%.2f)" % (s[len(s) // 2], s[0], s[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_dpm.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=BASE, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, _ = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    diffusion = b200mdm.SpacedDiffusion(use_timesteps=b200mdm.space_timesteps(BASE, STEPS),
                                        betas=gd.get_named_beta_schedule("cosine", BASE),
                                        model_mean_type=gd.ModelMeanType.START_X,
                                        model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE)
    n = diffusion.num_timesteps
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, model_kwargs={"y": y})
    samplers = {
        "ddim": lambda g: diffusion.ddim_sample_loop(cfg, shape, noise=x, noise_seed=1, use_graph=g, **kw),
        "dpm1": lambda g: diffusion.dpm_solver_sample_loop(cfg, shape, noise=x, order=1, use_graph=g, **kw),
        "dpm2": lambda g: diffusion.dpm_solver_sample_loop(cfg, shape, noise=x, order=2, use_graph=g, **kw),
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
        for _ in range(3):
            fn(True)
    torch.cuda.synchronize()
    warm = {k: [] for k in samplers}
    print("card:", card())
    for _ in range(a.runs):
        for k, fn in samplers.items():
            fn(True)                              # recaptures this sampler's step graph
            warm[k].append(timed(fn))             # warm graph
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in warm.items()}
    for k in samplers:
        print("%-5s B=%d T=%d L=%d %d steps (respaced from %d) CFG 2.5, %d runs: warm loop %s = %.3f ms/step, %.3f x DDIM"
              % (k, B, T, L, n, BASE, len(warm[k]), spread(warm[k]), med[k] / n, med[k] / med["ddim"]))

    from torch.profiler import ProfilerActivity, profile
    for k, fn in samplers.items():
        fn(False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(False)
            torch.cuda.synchronize()
        out = [(ev.device_time_total / 1e3, ev.count) for ev in prof.key_averages() if OUT_GEMM in ev.key]
        t_ms, cnt = sum(o[0] for o in out), sum(o[1] for o in out)
        print("%-5s output GEMM %.3f ms / %d launches = %.1f us per launch (plain launches, one loop)"
              % (k, t_ms, cnt, 1e3 * t_ms / max(cnt, 1)))


if __name__ == "__main__":
    main()
