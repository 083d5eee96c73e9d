"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/dip_longmem_small.npz by running the UNMODIFIED reference (via
oracle/ref_harness.py) on CPU with BERT text memories longer than 64 tokens:

    python -m oracle.gen_golden_longmem

Cases:
  dip_fwd_cfg, dip_ddpm   DiP (trans_dec + BERT memory, prefix completion): L=2, ctx 20 + pred 40, 3 steps, B=3,
                          Mt=150 with ragged masks (none / the last 60 tokens / a run in the middle and a tail),
                          guidance scales 7.5 / 2 / 1; a guided forward at t=1 and the DDPM loop
  bert_ddpm               the context_len = 0 BERT decoder: L=2, T=196, 3 steps, B=2, Mt=100 (none / the last 37
                          tokens padded), lengths 196 / 77, guidance 2.5 / 1
The reference's CPU decoder forward rounds differently with the number of intra-op threads, so the fixture is made,
and checked, with THREADS threads.  The inputs come from motion-diffusion-model_b200/synthetic.py (seeds below); this
module imports the reference harness only inside gen_longmem_small, so that the GPU tests can rebuild the inputs.
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")
OUT = os.path.join(ROOT, "tests", "golden")
THREADS = 8

DIP = dict(L=2, steps=3, B=3, ctx=20, pred=40, Mt=150, weights_seed=4, inputs_seed=13, dip_seed=14, lengths=[40, 33, 12],
           scales=[7.5, 2.0, 1.0])
BERT = dict(L=2, steps=3, B=2, T=196, Mt=100, weights_seed=5, inputs_seed=15, dip_seed=16, lengths=[196, 77],
            scales=[2.5, 1.0])


def dip_inputs():
    c = DIP
    enc, tmask, prefix = syn.synthetic_dip_inputs(c["B"], c["Mt"], c["ctx"], seed=c["dip_seed"])
    tmask[:] = False
    tmask[1, 90:] = True                   # right padding (the BERT case)
    tmask[2, 50:80] = True                 # a run in the middle (the C ABI takes any mask) and a tail
    tmask[2, 140:] = True
    inp = syn.synthetic_inputs(c["B"], nframes=c["pred"], steps=c["steps"], seed=c["inputs_seed"], lengths=c["lengths"],
                               scale=torch.tensor(c["scales"]))
    return inp, enc, tmask, prefix


def bert_inputs():
    c = BERT
    enc, tmask, _ = syn.synthetic_dip_inputs(c["B"], c["Mt"], 0, seed=c["dip_seed"])
    tmask[:] = False
    tmask[1, 63:] = True
    inp = syn.synthetic_inputs(c["B"], nframes=c["T"], steps=c["steps"], seed=c["inputs_seed"], lengths=c["lengths"],
                               scale=torch.tensor(c["scales"]))
    return inp, enc, tmask


def gen_longmem_small():
    from oracle import ref_harness as rh
    ns = rh.load_reference()
    threads = torch.get_num_threads()
    torch.set_num_threads(THREADS)
    try:
        out = {"meta": np.array(["DiP %s; BERT decoder %s; %d threads" % (DIP, BERT, THREADS)])}
        c = DIP
        args = rh.default_args(layers=c["L"], diffusion_steps=c["steps"], arch="trans_dec", text_encoder_type="bert",
                               context_len=c["ctx"], pred_len=c["pred"])
        model, diff = rh.build(args, state_dict=syn.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                                        seed=c["weights_seed"]))
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        inp, enc, tmask, prefix = dip_inputs()

        def y():
            return dict(mask=inp["mask"].clone(), lengths=inp["lengths"], text_embed=(enc, tmask), scale=inp["scale"],
                        prefix=prefix)
        with torch.no_grad():
            out["dip_fwd_cfg"] = cfg(inp["tape"][0], torch.full((c["B"],), 1, dtype=torch.long), y=y()).numpy()
            with rh.noise_tape(inp["tape"]):
                out["dip_ddpm"] = diff.p_sample_loop(cfg, (c["B"], 263, 1, c["pred"]), clip_denoised=False,
                                                     model_kwargs={"y": y()}).numpy()
        c = BERT
        args = rh.default_args(layers=c["L"], diffusion_steps=c["steps"], arch="trans_dec", text_encoder_type="bert")
        model, diff = rh.build(args, state_dict=syn.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                                        seed=c["weights_seed"]))
        cfg = ns.sampler_util.ClassifierFreeSampleModel(model)
        inp, enc, tmask = bert_inputs()
        yb = dict(mask=inp["mask"].clone(), lengths=inp["lengths"], text_embed=(enc, tmask), scale=inp["scale"])
        with torch.no_grad(), rh.noise_tape(inp["tape"]):
            out["bert_ddpm"] = diff.p_sample_loop(cfg, (c["B"], 263, 1, c["T"]), clip_denoised=False,
                                                  model_kwargs={"y": yb}).numpy()
    finally:
        torch.set_num_threads(threads)
    path = os.path.join(OUT, "dip_longmem_small.npz")
    np.savez_compressed(path, **out)
    print("dip_longmem_small.npz:", {k: v.shape for k, v in out.items() if k != "meta"}, os.path.getsize(path), "bytes")
    return out


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    gen_longmem_small()
