"""Time continuous batching of DiP chains (b200mdm.ContinuousChainSampler) at bench.py's dip shape: B = 128 slots,
pred_len 40, context_len 20, 8 layers, classifier-free guidance (scale 7.5), 10 DDPM steps, memories of 16 tokens,
196-frame requests (5 chunks), synthetic weights.  Prints the card and its power limit, then

  1. steady state, every slot busy: ms per step of the slot step graph against the uniform chain's step graph (Philox
     noise, same workspace shape), alternated in one process on two engines with the same weights;
  2. the cost of a hand-off (B hand-offs issued back to back at one boundary, wall time per hand-off), and the share of
     step time the boundaries take at steady state: B / n_steps boundaries per step on average (4 of 5 hand-offs that
     re-arm the chain, 1 the last hand-off; an admission per 5);
  3. a fixed-seed Poisson arrival trace at `load` x capacity (capacity = B / (5 x 10 x uniform step time)): throughput
     and p50 / p95 request latency (arrival to the motion's return) of ContinuousChainSampler against static batching
     (collect up to B arrived requests, then one AutoRegressiveSampler chain of B rows).

usage: python tools/time_continuous_chain.py [reps] [requests] [load]"""
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

B, PRED, CTX, STEPS, L, MT, FRAMES, C, SCALE = 128, 40, 20, 10, 8, 16, 196, 768, 7.5
CHUNKS = -(-FRAMES // PRED)


def default_args(**over):
    a = dict(dataset="humanml", unconstrained=False, latent_dim=512, layers=L, cond_mask_prob=0.1, arch="trans_dec",
             emb_trans_dec=False, text_encoder_type="bert", pos_embed_max_len=5000, mask_frames=True, pred_len=PRED,
             context_len=CTX, diffusion_steps=STEPS, noise_schedule="cosine", sigma_small=True, lambda_vel=0.0,
             lambda_rcxyz=0.0, lambda_fc=0.0)
    a.update(over)
    return SimpleNamespace(**a)


def build():
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(), SimpleNamespace(dataset=SimpleNamespace()))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=C, seed=0))
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


def inputs(n, seed):
    rng = np.random.default_rng(seed)
    tok = torch.from_numpy(rng.standard_normal((n, MT, C)).astype(np.float32)).cuda()
    pad = torch.zeros(n, MT, dtype=torch.bool)
    for i in range(n):
        pad[i, int(rng.integers(4, MT + 1)):] = True
    prefix = torch.from_numpy(rng.standard_normal((n, 263, 1, CTX)).astype(np.float32)).cuda()
    return tok, pad.cuda(), prefix


def steady(reps, k=STEPS - 2):
    cfg_u, model_u, diffusion = build()
    cfg_s, model_s, _ = build()
    tok, pad, prefix = inputs(B, 1)
    y = dict(prefix=prefix, text_embed=(tok.permute(1, 0, 2).contiguous(), pad), scale=torch.full((B,), SCALE, device="cuda"),
             mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"))
    shape = (B, 263, 1, PRED)
    diffusion.p_sample_loop(cfg_u, shape, clip_denoised=False, model_kwargs={"y": y}, noise_seed=3)   # conditioning, graph
    eu = model_u.engine()
    x = eu.philox_normal(shape, 3, 0, -1, "cuda")
    es = model_s.engine()
    state = {}

    def fresh():
        """A new slot session with every slot one step into its first chunk, outside the timed window."""
        cs = b200mdm.ContinuousChainSampler(diffusion, cfg_s, B, n_tokens=MT)
        for b in range(B):
            cs.submit(text_embed=(tok[b], pad[b]), prefix=prefix[b], length=FRAMES, scale=SCALE, seed=5)
        cs.step(1)
        state["cs"] = cs

    uni = lambda: eu.sample_loop_range(_lib.MODE_DDPM, STEPS - 1, k, x, None, None, 0, True)
    slot = lambda: es.slots_run(k, True)                   # k < STEPS - 1: no chunk ends inside the window
    timed(uni)
    fresh()
    timed(slot)
    tu, ts, th = [], [], []
    for _ in range(reps):
        tu.append(timed(uni) / k)
        fresh()
        ts.append(timed(slot) / k)
        # every slot at its first boundary: B hand-offs back to back (wall time, host enqueue included)
        es.slots_run(STEPS - 1 - k, True)
        cs = state["cs"]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in range(B):
            cs.scheduler.engine.slot_handoff(b, cs.scheduler.occupant[b], 0)
        torch.cuda.synchronize()
        th.append((time.perf_counter() - t0) * 1000.0 / B)
    return [float(np.median(v)) for v in (tu, ts, th)] + [tu, ts, th]


def trace(n_req, load, step_ms, seed=0):
    cfg, model, diffusion = build()
    rng = np.random.default_rng(seed)
    capacity = B / (CHUNKS * STEPS * step_ms / 1000.0)     # requests / s
    arrivals = np.cumsum(rng.exponential(1.0 / (load * capacity), n_req))
    tok, pad, prefix = inputs(n_req, seed + 1)
    res = {}

    # continuous batching: every step boundary admits what has arrived
    cs = b200mdm.ContinuousChainSampler(diffusion, cfg, B, n_tokens=MT)
    cs.submit(text_embed=(tok[0], pad[0]), prefix=prefix[0], length=FRAMES, scale=SCALE, seed=1)   # warm-up: capture
    cs.drain()
    torch.cuda.synchronize()
    t0, nxt, done = time.perf_counter(), 0, {}
    while len(done) < n_req:
        now = time.perf_counter() - t0
        while nxt < n_req and arrivals[nxt] <= now:
            cs.submit(text_embed=(tok[nxt], pad[nxt]), prefix=prefix[nxt], length=FRAMES, scale=SCALE, seed=7,
                      sample_index=nxt)
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

    # static batching: collect up to B arrived requests, then one chain of B rows
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=False)
    ar = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, required_frames=FRAMES)

    def y(idx):
        i = torch.as_tensor(np.resize(idx, B), device="cuda")
        return dict(prefix=prefix[i], text_embed=(tok[i].permute(1, 0, 2).contiguous(), pad[i]),
                    scale=torch.full((B,), SCALE, device="cuda"), mask=torch.ones(B, 1, 1, PRED, dtype=torch.bool, device="cuda"))
    ar.sample(cfg, (B, 263, 1, PRED), clip_denoised=False, model_kwargs={"y": y([0])}, noise_seed=7)
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
        ar.sample(cfg, (B, 263, 1, PRED), clip_denoised=False, model_kwargs={"y": y(idx)}, noise_seed=7,
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
    n_req = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
    load = float(sys.argv[3]) if len(sys.argv) > 3 else 0.9
    torch.cuda.set_device(0)
    print("card: %s" % card())
    tu, ts, th, all_u, all_s, all_h = steady(reps)
    print("steady state, B = %d, pred_len %d + context %d, L = %d, CFG, Mt = %d: uniform chain step %.3f ms, slot step "
          "%.3f ms (medians of %d; uniform %s, slot %s)" % (B, PRED, CTX, L, MT, tu, ts, reps,
                                                           ["%.3f" % v for v in all_u], ["%.3f" % v for v in all_s]))
    per_step = B / STEPS                                   # boundaries per step with staggered slots
    print("hand-off: %.4f ms wall each (medians of %d: %s); %.1f boundaries per step at steady state: %.3f ms, %.1f%% of "
          "a step" % (th, reps, ["%.4f" % v for v in all_h], per_step, per_step * th,
                      100.0 * per_step * th / (ts + per_step * th)))
    print("Poisson trace: %d requests of %d frames at %.2f x capacity (%.0f requests/s from the uniform step):"
          % (n_req, FRAMES, load, B / (CHUNKS * STEPS * tu / 1000.0)))
    trace(n_req, load, tu)


if __name__ == "__main__":
    main()
