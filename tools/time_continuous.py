"""Time continuous batching (b200mdm.ContinuousSampler) at bench.py's c2 shape: B = 64 slots, T = 196, 8 layers,
classifier-free guidance, 50 DDPM steps, synthetic weights.  Prints the card and its power limit, then

  1. steady state, every slot busy: ms per step of the slot step graph against the uniform step graph (Philox noise,
     same workspace shape), alternated in one process on two engines with the same weights;
  2. a fixed-seed Poisson arrival trace at `load` x capacity (capacity = B / (50 x uniform step time)): throughput and
     p50 / p95 request latency (arrival to the motion's return) of ContinuousSampler against static batching (collect up
     to B arrived requests, then one p_sample_loop of B rows).

usage: python tools/time_continuous.py [reps] [requests] [load]"""
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200mdm  # noqa: E402
from b200mdm import _lib  # noqa: E402

B, T, STEPS, L = 64, 196, 50, 8


def default_args(**over):
    a = dict(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1, arch="trans_enc",
             emb_trans_dec=False, text_encoder_type="clip", pos_embed_max_len=5000, mask_frames=True, pred_len=0,
             context_len=0, diffusion_steps=STEPS, noise_schedule="cosine", sigma_small=True, lambda_vel=0.0,
             lambda_rcxyz=0.0, lambda_fc=0.0)
    a.update(over)
    return SimpleNamespace(**a)


def build():
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(), SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(num_layers=L, seed=0))
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:   # the numbers below are still printed, without the card's limit
        return "nvidia-smi unavailable (%s)" % exc


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def steady(reps, k=40):
    cfg_u, model_u, diffusion = build()
    cfg_s, model_s, _ = build()
    g = torch.Generator(device="cuda").manual_seed(1)
    te = torch.randn(1, B, 512, device="cuda", generator=g)
    y = dict(mask=torch.ones(B, 1, 1, T, dtype=torch.bool, device="cuda"), lengths=torch.full((B,), T, device="cuda"),
             text_embed=te, scale=torch.full((B,), 2.5, device="cuda"))
    shape = (B, 263, 1, T)
    diffusion.p_sample_loop(cfg_u, shape, clip_denoised=False, model_kwargs={"y": y}, noise_seed=3)   # conditioning, graph
    eu = model_u.engine()
    x = eu.philox_normal(shape, 3, 0, -1, "cuda")
    es = model_s.engine()

    def fresh():
        """A new slot session with every slot busy (49 steps left), outside the timed window."""
        cs = b200mdm.ContinuousSampler(diffusion, cfg_s, B, T)
        for b in range(B):
            cs.submit(text_embed=te[0, b], scale=2.5, seed=5)
        cs.step(1)
        return cs

    uni = lambda: eu.sample_loop_range(_lib.MODE_DDPM, STEPS - 1, k, x, None, None, 0, True)
    slot = lambda: es.slots_run(k, True)                   # k < 49: no slot finishes inside the window
    timed(uni)
    fresh()
    timed(slot)
    tu, ts = [], []
    for _ in range(reps):
        tu.append(timed(uni) / k)
        fresh()
        ts.append(timed(slot) / k)
    return float(np.median(tu)), float(np.median(ts)), tu, ts


def trace(n_req, load, step_ms, seed=0):
    cfg, model, diffusion = build()
    rng = np.random.default_rng(seed)
    capacity = B / (STEPS * step_ms / 1000.0)              # requests / s
    arrivals = np.cumsum(rng.exponential(1.0 / (load * capacity), n_req))
    te = torch.from_numpy(rng.standard_normal((n_req, 512)).astype(np.float32)).cuda()
    lengths = rng.integers(40, T + 1, n_req)
    res = {}

    # continuous batching: every step boundary admits what has arrived
    cs = b200mdm.ContinuousSampler(diffusion, cfg, B, T)
    cs.submit(text_embed=te[0], scale=2.5, seed=1, length=T)       # warm-up request: capture the slot graph
    cs.drain()
    torch.cuda.synchronize()
    t0, nxt, done = time.perf_counter(), 0, {}
    while len(done) < n_req:
        now = time.perf_counter() - t0
        while nxt < n_req and arrivals[nxt] <= now:
            cs.submit(text_embed=te[nxt], length=int(lengths[nxt]), scale=2.5, seed=7, sample_index=nxt)
            nxt += 1
        if cs.active == 0 and cs.pending == 0:
            time.sleep(max(0.0, arrivals[nxt] - now))
            continue
        out = cs.step(1)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        for rid, _ in out:
            done[rid - 1] = t                                      # ids after the warm-up request start at 1
    res["continuous"] = (done, time.perf_counter() - t0)

    # static batching: collect up to B arrived requests, then one loop of B rows
    y = lambda idx: dict(
        mask=(torch.arange(T, device="cuda")[None, :] < torch.as_tensor(np.resize(lengths[idx], B), device="cuda")[:, None]
              ).reshape(B, 1, 1, T),
        lengths=torch.as_tensor(np.resize(lengths[idx], B), device="cuda"),
        text_embed=te[torch.as_tensor(np.resize(idx, B), device="cuda")].unsqueeze(0), scale=torch.full((B,), 2.5, device="cuda"))
    diffusion.p_sample_loop(cfg, (B, 263, 1, T), clip_denoised=False, model_kwargs={"y": y([0])}, noise_seed=7)
    torch.cuda.synchronize()
    t0, nxt, done = time.perf_counter(), 0, {}
    while len(done) < n_req:
        now = time.perf_counter() - t0
        if nxt < n_req and arrivals[nxt] > now:
            time.sleep(arrivals[nxt] - now)
            continue
        idx = []
        while nxt < n_req and arrivals[nxt] <= now and len(idx) < B:
            idx.append(nxt)
            nxt += 1
        diffusion.p_sample_loop(cfg, (B, 263, 1, T), clip_denoised=False, model_kwargs={"y": y(idx)}, noise_seed=7,
                                sample_index_base=idx[0])
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        for i in idx:
            done[i] = t
    res["static"] = (done, time.perf_counter() - t0)
    for name, (done, wall) in res.items():
        lat = np.array([done[i] - arrivals[i] for i in range(n_req)]) * 1000.0
        print("  %-10s  %7.1f motions/s   latency p50 %7.1f ms   p95 %7.1f ms   (wall %.2f s)"
              % (name, n_req / wall, np.percentile(lat, 50), np.percentile(lat, 95), wall))


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    n_req = int(sys.argv[2]) if len(sys.argv) > 2 else 512
    load = float(sys.argv[3]) if len(sys.argv) > 3 else 0.9
    torch.cuda.set_device(0)
    print("card: %s" % card())
    tu, ts, all_u, all_s = steady(reps)
    print("steady state, B = %d, T = %d, L = %d, CFG: uniform step %.3f ms, slot step %.3f ms (medians of %d; uniform %s, "
          "slot %s)" % (B, T, L, tu, ts, reps, ["%.3f" % v for v in all_u], ["%.3f" % v for v in all_s]))
    print("Poisson trace: %d requests at %.2f x capacity (%.0f requests/s from the uniform step), lengths 40..%d:"
          % (n_req, load, B / (STEPS * tu / 1000.0), T))
    trace(n_req, load, tu)


if __name__ == "__main__":
    main()
