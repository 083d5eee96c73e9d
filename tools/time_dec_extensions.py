"""Time the sampling extensions on the BERT decoder with context_len 0 (humanml_trans_dec_512_bert): 8 layers, B = 64
motions of 196 frames, a 24-token text memory (a typical HumanML3D caption under DistilBERT), 50 DDPM steps on the
engine's Philox stream and its step graph.  Plain classifier-free guidance (scale 2.5), handshakes (h = 20, four windows
per motion), joint-position control (pelvis and wrists, step size 2e-4) at K = 1, 10 and 50 guidance iterations per
step, and multi-prompt guidance at K = 1 (w = 2.5), 2 and 3 prompts run in turn on one
engine (--runs rounds); each turn starts with one untimed loop that recaptures its step graph, then times one warm loop
with CUDA events.  The card's name, power limit and SM clock are read in the same process.

    python tools/time_dec_extensions.py [--runs 5]
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

B, T, L, STEPS, SCALE, MT, H = 64, 196, 8, 50, 2.5, 24, 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_dec_extensions.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_dec", emb_trans_dec=False, text_encoder_type="bert", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=768, seed=0))
    model = model.to("cuda").eval()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    g = torch.Generator().manual_seed(1)

    def prompt(seed):
        enc, tmask, _ = b200mdm.synthetic_dip_inputs(B, MT, 0, seed=seed)
        tmask[:] = torch.arange(MT)[None, :] >= torch.randint(8, MT + 1, (B, 1), generator=g)   # right padding
        return enc.cuda(), tmask.cuda()

    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda())
    plain = dict(base, text_embed=prompt(2), scale=torch.full((B,), SCALE, device="cuda"))
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    ms = torch.zeros(B, dtype=torch.bool)
    ms[::4] = True
    ys = {"CFG": (cfg, plain),
          "handshake": (b200mdm.HandshakeSampleModel(cfg, H), dict(plain, motion_start=ms.cuda()))}
    mean, std = torch.zeros(263), torch.ones(263)
    target = torch.randn(B, 22, 3, T, generator=g) * 0.5
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    weight[:, 20:22, ::49] = 1.0
    for iters in (1, 10, 50):
        ys["joint K=%d" % iters] = (b200mdm.JointControlSampleModel(cfg, mean, std, 2e-4, iters),
                                    dict(plain, joint_target=target.cuda(), joint_weight=weight.cuda()))
    mp = b200mdm.MultiPromptSampleModel(model)
    for K in (1, 2, 3):
        w = torch.full((B, K, 1, 1), SCALE) if K == 1 else torch.rand(B, K, 263, T, generator=g) * SCALE
        ys["multi K=%d" % K] = (mp, dict(base, prompt_embed=[prompt(2 + k) for k in range(K)], prompt_weight=w.cuda()))
    kw = dict(clip_denoised=False, noise_seed=1)
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
        print("%-11s loop %s, per step %.3f ms, %+.3f ms per step over CFG (x%.2f)"
              % (k, spread(v), med / STEPS, (med - base_ms) / STEPS, med / base_ms))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
