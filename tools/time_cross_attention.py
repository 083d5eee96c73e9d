"""Time the DiP cross-attention core against the text-memory length Mt (CUDA events, after warm-up, median of reps):
  * the core alone at the engine's launch (2 x 64 samples = B 64 with guidance, 4 heads), S = 60 and S = 196:
    cross_attention_kernel<MAX_NT> for Mt <= 64, cross_attention_long_kernel above;
  * one DiP sampling step (8 layers, B = 64, guidance 7.5, 20 + 40 frames) from a 10-step fused loop.
Prints the card name and power limit of the same run."""
import ctypes
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200mdm  # noqa: E402
from b200mdm import _lib as L  # noqa: E402

MTS = [16, 64, 65, 128, 256, 512]


def timed(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def core_us(n, S, Mt, inner=50):
    lib = L.load()
    d, ld = 512, 8 * 1024
    g = torch.Generator(device="cuda").manual_seed(Mt + S)
    q = torch.randn(n * S, d, device="cuda", generator=g).half()
    kv = torch.randn(n * Mt, ld, device="cuda", generator=g).half()
    mask = torch.zeros(n, Mt, dtype=torch.uint8, device="cuda")
    mask[1::2, Mt // 2:] = 1
    out = torch.empty(n * S, 2 * d, device="cuda", dtype=torch.float16)
    kv7 = ctypes.c_void_p(kv.data_ptr() + 2 * 7 * 1024)              # layer 7's k | v columns
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        for _ in range(inner):
            L.check(lib.b200mdm_test_cross_attention(ctypes.c_void_p(q.data_ptr()), kv7, ctypes.c_void_p(mask.data_ptr()),
                                                     ctypes.c_void_p(out.data_ptr()), n, S, Mt, ld, st))
    return timed(run) * 1e3 / inner


def dip_step_ms(Mt, B=64, steps=10):
    ctx, pred = 20, 40
    args = SimpleNamespace(dataset="humanml", unconstrained=False, latent_dim=512, layers=8, cond_mask_prob=0.1,
                           arch="trans_dec", emb_trans_dec=False, text_encoder_type="bert", pos_embed_max_len=5000,
                           mask_frames=True, pred_len=pred, context_len=ctx, diffusion_steps=steps, noise_schedule="cosine",
                           sigma_small=True, lambda_vel=0.0, lambda_rcxyz=0.0, lambda_fc=0.0)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=8, cond_dim=768, seed=23))
    model.to("cuda").eval()
    cfg = b200mdm.ClassifierFreeSampleModel(model)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, ctx, seed=35)
    y = dict(mask=torch.ones(B, 1, 1, pred, dtype=torch.bool, device="cuda"), lengths=torch.full((B,), pred, device="cuda"),
             text_embed=(enc.cuda(), tmask.cuda()), prefix=prefix.cuda(), scale=torch.full((B,), 7.5, device="cuda"))
    g = torch.Generator(device="cuda").manual_seed(1)
    shape = (B, 263, 1, pred)
    xT = torch.randn(*shape, device="cuda", generator=g)
    tape = torch.randn(steps, *shape, device="cuda", generator=g)
    ms = timed(lambda: diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y},
                                               noise_tape=tape), reps=10)
    return ms / steps


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(0), "|", q.splitlines()[0] if q else "nvidia-smi unavailable")
    print("%6s %22s %22s %18s" % ("Mt", "core S=60 (us)", "core S=196 (us)", "DiP step (ms)"))
    for Mt in MTS:
        print("%6d %22.2f %22.2f %18.3f" % (Mt, core_us(128, 60, Mt), core_us(128, 196, Mt), dip_step_ms(Mt)), flush=True)


if __name__ == "__main__":
    main()
