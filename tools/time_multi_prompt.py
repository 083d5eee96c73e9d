"""Time multi-prompt guidance (MultiPromptSampleModel) at the bench's encoder shape: trans_enc, 8 layers, B = 64 motions
of 196 frames, 50 DDPM steps on the engine's Philox stream and its step graph.  ClassifierFreeSampleModel at scale 2.5
and the composed path at K = 1 (w = 2.5), 2 and 3 run in turn on one engine (--runs rounds); each turn starts with one
untimed loop that recaptures its step graph, then times one warm loop with CUDA events.  A separate profiled loop per
configuration (torch.profiler, CUDA activity) gives the per-step time of the kernels the composition changes: the blend,
the output GEMM (the EpiOut instantiation) and compose_step_kernel, which writes nothing the CFG path reads, so the
output GEMM's extra rows and the raw-x0 round trip are those two kernels' time over the CFG path's output GEMM.  The
card's name, power limit and SM clock are read in the same process.

    python tools/time_multi_prompt.py [--runs 5]
"""
import argparse
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200mdm  # noqa: E402
from time_dpm import card, spread  # noqa: E402

B, T, L, STEPS, SCALE = 64, 196, 8, 50, 2.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_multi_prompt.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    model = model.to("cuda").eval()
    cfg, mp = b200mdm.ClassifierFreeSampleModel(model), b200mdm.MultiPromptSampleModel(model)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda())
    g = torch.Generator().manual_seed(1)
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, noise_seed=1)
    ys = {"CFG": (cfg, dict(base, text_embed=inp["text_embed"].cuda(), scale=torch.full((B,), SCALE, device="cuda")))}
    for K in (1, 2, 3):
        w = torch.full((B, K, 1, 1), SCALE) if K == 1 else torch.rand(B, K, 263, T, generator=g) * SCALE
        ys["K=%d" % K] = (mp, dict(base, prompt_embed=(torch.randn(K, B, 512, generator=g) * 0.5).cuda(),
                                   prompt_weight=w.cuda()))
    loops = {k: (lambda m, y: lambda: diffusion.p_sample_loop(m, shape, noise=x, model_kwargs={"y": y}, **kw))(*v)
             for k, v in ys.items()}

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
    base_ms = sorted(t["CFG"])[len(t["CFG"]) // 2]
    for k, v in t.items():
        med = sorted(v)[len(v) // 2]
        print("%-4s loop %s, per step %.3f ms, %+.3f ms per step over CFG (x%.2f)"
              % (k, spread(v), med / STEPS, (med - base_ms) / STEPS, med / base_ms))
    from torch.profiler import ProfilerActivity, profile
    for k, fn in loops.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tot = {"blend": 0.0, "output GEMM": 0.0, "compose": 0.0, "all": 0.0}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            tot["all"] += us
            if "blend_split" in ev.name:
                tot["blend"] += us
            elif "compose_step" in ev.name:           # (its signature names EpiOutParams: matched first)
                tot["compose"] += us
            elif "EpiOut" in ev.name:
                tot["output GEMM"] += us
        print("%-4s per step (profiled): " % k + ", ".join("%s %.1f us" % (n, v / STEPS) for n, v in tot.items()))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
