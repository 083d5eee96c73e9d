"""Time DoubleTake's two takes at the headline shape: trans_enc, 8 layers, 64 windows of 196 frames as 8 motions of 8,
h = 20, CFG 2.5, 50 DDIM steps on the engine's Philox noise stream.  Take 1 is the HandshakeSampleModel loop; take 2 is
refine_transitions with m = 10 (56 transitions of 40 frames) at k = 25, gather, stitch and paste included.  Both are
timed with a host clock around work that ends in a device synchronise, alternately (--runs rounds, after warm-up).  The
card's name, power limit and SM clock are read in the same process.  A separate torch.profiler pass reports the output
GEMM's (EpiOut<OutStep>) device time per launch on the transition batch with a soft weight, a bool mask and no
inpainting.

    python tools/time_double_take.py [--runs 7]
"""
import argparse
import os
import sys
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200mdm  # noqa: E402
from time_dpm import card, spread  # noqa: E402

B, T, L, STEPS, H, PER, M, K = 64, 196, 8, 50, 20, 8, 10, 25


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_double_take.py needs a GPU")
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
    kw = dict(clip_denoised=False, eta=0.0)
    windows = diffusion.ddim_sample_loop(hs, shape, model_kwargs={"y": y}, noise_seed=1, **kw)
    loops = {
        "take1": lambda: diffusion.ddim_sample_loop(hs, shape, model_kwargs={"y": y}, noise_seed=1, **kw),
        "take2": lambda: b200mdm.refine_transitions(diffusion.ddim_sample_loop, cfg, windows, {"y": y}, H, M, K,
                                                    noise_seed=2, **kw),
    }

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0)

    print("library:", b200mdm._lib.LIB_PATH)
    lay = b200mdm.transition_layout(B, T, H, M, y["lengths"], y["motion_start"])
    n, Lt = lay["pairs"].shape[0], lay["weight"].shape[0]
    print("take 2: %d transitions of %d frames, %d of %d steps" % (n, Lt, STEPS - K, STEPS))
    for fn in loops.values():                     # warm-up: workspaces, clocks
        for _ in range(3):
            fn()
    print("card:", card())
    res = {k: [] for k in loops}
    for _ in range(a.runs):
        for k, fn in loops.items():
            res[k].append(timed(fn))
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    for k in loops:
        print("%-6s %d runs: %s ms, median %.3f ms, %.4f x take 1" % (k, len(res[k]), spread(res[k]), med[k],
                                                                      med[k] / med["take1"]))
    # profiler pass (separate from the timed runs): the output GEMM per launch on the transition batch
    from torch.profiler import ProfilerActivity, profile
    sw, sf = torch.from_numpy(lay["src_window"]).cuda(), torch.from_numpy(lay["src_frame"]).cuda()
    x_init = windows[sw, :, :, sf].permute(0, 2, 3, 1).contiguous()
    w = torch.from_numpy(lay["weight"]).cuda().view(1, 1, 1, Lt).expand_as(x_init).contiguous()
    bidx = torch.from_numpy(lay["pairs"][:, 1]).cuda()
    yt = dict(text_embed=y["text_embed"][:, bidx], scale=y["scale"][bidx])
    variants = dict(weight=dict(yt, inpainting_weight=w, inpainted_motion=x_init),
                    mask=dict(yt, inpainting_mask=w >= 0.5, inpainted_motion=x_init), none=yt)
    for k, yy in variants.items():
        def run():
            diffusion.ddim_sample_loop(cfg, tuple(x_init.shape), model_kwargs={"y": yy}, skip_timesteps=K, init_image=x_init,
                                       noise_seed=2, **kw)
        run()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "EpiOut" in e.key]
        tot, cnt = sum(e.device_time_total for e in ev), sum(e.count for e in ev)
        print("%-6s output GEMM (EpiOut<OutStep>) on [%d, 263, 1, %d]: %d launches, %.2f us per launch"
              % (k, n, Lt, cnt, tot / max(cnt, 1)))


if __name__ == "__main__":
    main()
