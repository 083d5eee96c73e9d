"""Time chained windows (HandshakeSampleModel) against the plain guided model at BASELINE config 2's shape: trans_enc,
8 layers, 64 windows of 196 frames as 8 motions of 8, h = 20, CFG 2.5, 50 DDIM steps, on the engine's Philox noise
stream and its step graph.  The two loops run alternately on the same engine (--runs rounds); each turn starts with one
loop that recaptures its step graph (untimed), then times one warm replay with CUDA events.  The card's name, power
limit and SM clock are read in the same process.  A separate torch.profiler pass then reports blend_split_kernel's
device time per launch in each loop.

    python tools/time_handshake.py [--runs 7]
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

B, T, L, STEPS, H, PER = 64, 196, 8, 50, 20, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_handshake.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    hs = b200mdm.HandshakeSampleModel(cfg, H)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda(), motion_start=(torch.arange(B) % PER == 0).cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, eta=0.0, model_kwargs={"y": y}, noise_seed=1)
    loops = {
        "plain": lambda: diffusion.ddim_sample_loop(cfg, shape, noise=x, **kw),
        "handshake": lambda: diffusion.ddim_sample_loop(hs, shape, noise=x, **kw),
    }

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    print("library:", b200mdm._lib.LIB_PATH)
    chained = int((~y["motion_start"]).sum())
    print("frame rows that read a second row pair: %d of %d (%.1f %%)" % (2 * chained * H, B * T, 100.0 * 2 * chained * H / (B * T)))
    for fn in loops.values():                     # warm-up: workspace, clocks
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    warm = {k: [] for k in loops}
    print("card:", card())
    for _ in range(a.runs):
        for k, fn in loops.items():
            fn()                                  # recapture (the other loop's graph was the workspace's)
            warm[k].append(timed(fn))
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in warm.items()}
    for k in loops:
        print("%-9s B=%d T=%d L=%d DDIM %d steps CFG 2.5, %d runs: warm loop %s = %.3f ms/step, %.4f x plain"
              % (k, B, T, L, STEPS, len(warm[k]), spread(warm[k]), med[k] / STEPS, med[k] / med["plain"]))
    # profiler pass (separate from the timed runs): blend_split_kernel per launch
    from torch.profiler import ProfilerActivity, profile
    for k, fn in loops.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "blend_split_kernel" in e.key]
        tot = sum(e.device_time_total for e in ev)
        cnt = sum(e.count for e in ev)
        allk = sum(e.device_time_total for e in prof.key_averages() if e.device_type.name == "CUDA")
        print("%-9s blend_split_kernel: %d launches, %.2f us per launch, %.2f %% of the loop's kernel time"
              % (k, cnt, tot / max(cnt, 1), 100.0 * tot / max(allk, 1e-9)))


if __name__ == "__main__":
    main()
