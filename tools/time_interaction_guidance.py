"""Time the interaction terms of joint-position control at the headline shape: trans_enc, 8 layers, B = 64 motions of
196 frames, CFG 2.5, 50 DDPM steps on the engine's Philox stream and its step graph, K = 10.  Five loops run in turn
on one engine (--runs alternated rounds): unguided, the scene-guided loop (the pelvis on every frame, contact weight 4,
floor weight 2, derived contacts, obstacles of weight 4 and margin 0.3 from the SDF of three discs and a wall box on a
161 x 161 grid of 5 cm), and the same with the interaction terms in scenes of C = 2, 4 and 8 characters (weight 4,
margin 0.3, characters 0.5 m apart, two reach rows per scene); each turn starts with one untimed loop that recaptures
its step graph, then times one warm loop with CUDA events.  The card's name, power limit and SM clock are read in the
same process.

    python tools/time_interaction_guidance.py [--runs 5]
"""
import argparse
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200mdm  # noqa: E402
from oracle import joint_control_oracle as jo  # noqa: E402
from oracle import ric_oracle  # noqa: E402
from time_dpm import card, spread  # noqa: E402

B, T, L, STEPS, STEP, K, CW, FW, OW, R = 64, 196, 8, 50, 2e-5, 10, 4.0, 2.0, 4.0, 0.3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_interaction_guidance.py needs a GPU")
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1,
                           arch="trans_enc", emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=0, context_len=0, diffusion_steps=STEPS, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=0, seed=10)
    mean, std = jo.motion_stats(263)
    g = torch.Generator().manual_seed(3)
    data = (torch.randn(B, 263, T, generator=g) * 0.5 * std[None, :, None] + mean[None, :, None]).permute(0, 2, 1)
    target = ric_oracle.recover_from_ric(data, 22).permute(0, 2, 3, 1).contiguous()
    weight = torch.zeros(B, 22, T)
    weight[:, 0] = 1.0
    base = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(),
                scale=inp["scale"].cuda())
    joint = dict(base, joint_target=target.cuda(), joint_weight=weight.cuda())
    shape = (B, 263, 1, T)
    x = inp["tape"][0].cuda()
    kw = dict(contact_weight=CW, floor_weight=FW, obstacle_weight=OW, obstacle_margin=R)
    o, c, n = (-4.0, -4.0), 0.05, 161
    sdf = b200mdm.SceneGrid.from_shapes((n, n), o, c, discs=[(0.0, 0.5, 0.4), (1.0, 1.0, 0.3), (-0.8, -0.6, 0.3)],
                                        boxes=[(-2.0, 1.5, 2.0, 1.7)])
    scene = dict(joint, obstacle_sdf=sdf)

    def loop(m, y):
        return lambda: diffusion.p_sample_loop(m, shape, noise=x, clip_denoised=False, model_kwargs={"y": y}, noise_seed=1)
    loops = {"unguided": loop(cfg, base),
             "scene": loop(b200mdm.JointControlSampleModel(cfg, mean, std, STEP, K, **kw), scene)}
    for C in (2, 4, 8):
        pl = torch.zeros(B, 3)
        pl[:, 0] = 0.5 * (torch.arange(B) % C).float()
        pl[:, 2] = 0.3 * (torch.arange(B) % C).float()
        rows = torch.tensor([[0, 20, 1, 21], [1, 4, 0, 10]])
        inter = dict(scene, scene_placement=pl.cuda(), interaction_pairs=rows, interaction_reach=torch.tensor([0.05, 0.1]),
                     interaction_pair_weight=torch.ones(2, T).cuda())
        jc = b200mdm.JointControlSampleModel(cfg, mean, std, STEP, K, characters=C, interaction_weight=OW,
                                             interaction_margin=R, **kw)
        loops["C=%d" % C] = loop(jc, inter)

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
    ref = sorted(t["scene"])[len(t["scene"]) // 2]
    for k, v in t.items():
        med = sorted(v)[len(v) // 2]
        print("%-9s loop %s, per step %.3f ms, %+.3f ms per step over the scene-guided loop" % (k, spread(v), med / STEPS,
                                                                                              (med - ref) / STEPS))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
