"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/mixed_t_small.npz by running the UNMODIFIED reference
(/root/reference, via oracle/ref_harness.py) on CPU:

    python -m oracle.gen_golden_mixed_t

The reference's p_sample and ddim_sample are per sample: t is a [B] tensor, _extract_into_tensor gathers one schedule
row per sample and the model embeds each sample's own timestep.  This fixture pins one such step with a different
schedule index in every row: trans_enc L=2, 8 steps, B=4, T=24, ragged lengths, per-sample scales (one of them 0),
classifier-free guidance, t = (7, 0, 3, 5), a given eps, clip_denoised=False; p_sample, and ddim_sample at eta 0 and
0.5.  Each entry holds the step's sample and pred_xstart.
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
L, STEPS, B, T = 2, 8, 4, 24
LENGTHS, SCALES, TS = [24, 17, 5, 12], [2.5, 1.0, 7.5, 0.0], [7, 0, 3, 5]


def inputs():
    """The step's inputs (tests/test_continuous_gpu.py rebuilds the same): synthetic_inputs' x_T as x, its first eps."""
    inp = syn.synthetic_inputs(B, nframes=T, steps=STEPS, seed=21, lengths=LENGTHS, scale=torch.tensor(SCALES))
    return inp, inp["tape"][0], inp["tape"][1]


def main():
    # the harness loads the reference, which exists only where the fixture is made: the tests import inputs() alone
    from oracle import ref_harness as rh
    from oracle.gen_golden import _y
    args = rh.default_args(layers=L, diffusion_steps=STEPS)
    model, diff = rh.build(args, state_dict=syn.synthetic_state_dict(num_layers=L, seed=1))
    cfg = rh.load_reference().sampler_util.ClassifierFreeSampleModel(model)
    inp, x, eps = inputs()
    t = torch.tensor(TS, dtype=torch.long)
    out = {"meta": np.array(["L=%d steps=%d B=%d T=%d weights_seed=1 inputs_seed=21 lengths=%s scales=%s t=%s"
                             % (L, STEPS, B, T, LENGTHS, SCALES, TS)])}
    with torch.no_grad():
        for name, eta in (("ddpm", None), ("ddim_eta0", 0.0), ("ddim_eta0.5", 0.5)):
            with rh.noise_tape([eps]):
                if eta is None:
                    o = diff.p_sample(cfg, x, t, clip_denoised=False, model_kwargs={"y": _y(inp)})
                else:
                    o = diff.ddim_sample(cfg, x, t, clip_denoised=False, model_kwargs={"y": _y(inp)}, eta=eta)
            out[name + "_sample"] = o["sample"].numpy()
            out[name + "_pred_xstart"] = o["pred_xstart"].numpy()
    np.savez_compressed(os.path.join(OUT, "mixed_t_small.npz"), **out)
    print("mixed_t_small.npz:", {k: v.shape for k, v in out.items() if k != "meta"})


if __name__ == "__main__":
    main()
