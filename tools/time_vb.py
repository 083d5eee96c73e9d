"""Time the variational-bound loop (calc_bpd_loop) against the DDPM loop (p_sample_loop) at BASELINE config 2's shape:
trans_enc, 8 layers, B=64, 196 frames, CFG 2.5, a 50-step cosine schedule, both on the engine's Philox noise stream and
its step graph.  The two loops run alternately on the same engine (--runs rounds); each turn starts with one loop that
recaptures its step graph (untimed), then times one warm replay with CUDA events.  The card's name, power limit and SM
clock are read in the same process.  Launches per step come from the engine's launch counter.

    python tools/time_vb.py [--runs 7]
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

B, T, L, STEPS = 64, 196, 8, 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_vb.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    eng = model.engine()
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
             scale=inp["scale"].cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(clip_denoised=False, model_kwargs={"y": y}, noise_seed=1)
    loops = {
        "ddpm": lambda: diffusion.p_sample_loop(cfg, shape, noise=x, **kw),
        "bound": lambda: diffusion.calc_bpd_loop(cfg, x, **kw),
    }

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    print("library:", b200mdm._lib.LIB_PATH)
    for fn in loops.values():                     # warm-up: workspace, clocks
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    launches = {}
    for k, fn in loops.items():
        fn()                                      # recapture
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        fn()
        torch.cuda.synchronize()
        launches[k] = eng.launch_count(reset=True)
    warm = {k: [] for k in loops}
    print("card:", card())
    for _ in range(a.runs):
        for k, fn in loops.items():
            fn()
            warm[k].append(timed(fn))
    print("card:", card())
    med = {k: sorted(v)[len(v) // 2] for k, v in warm.items()}
    for k in loops:
        print("%-5s B=%d T=%d L=%d %d steps CFG 2.5, %d runs: warm loop %s = %.3f ms/step, %.3f x DDPM; %d launches per "
              "loop (%.2f per step)" % (k, B, T, L, STEPS, len(warm[k]), spread(warm[k]), med[k] / STEPS,
                                        med[k] / med["ddpm"], launches[k], launches[k] / STEPS))


if __name__ == "__main__":
    main()
