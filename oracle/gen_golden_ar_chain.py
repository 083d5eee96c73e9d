"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/dip_ar_small.npz by running the UNMODIFIED reference's own
AutoRegressiveSampler (utils/sampler_util.py:41-81) with its p_sample_loop on CPU, every draw taken from a noise tape
(oracle/ref_harness.py), in the build container:

    python -m oracle.gen_golden_ar_chain

The reference's text encoder is third-party; both sides get TableBert, which maps each prompt to seeded BERT-shaped
features, so the fixture pins the chain itself: how many chunks, which frames become the next prefix, the
include_prefix offset, the crop at required_frames and the per-chunk x_T and eps order.

Cases (DiP L=2, ctx 20 + pred 40, 3 DDPM steps per chunk, B=3, Mt=7, per-sample scales, ragged lengths):
  dyn196   a prompt per chunk (y['text'] a list of lists), include_prefix, 196 frames = 5 chunks, the last cropped
  static100  one prompt per sample for every chunk, no prefix in the output, 100 frames = 3 chunks, the last cropped
Each case stores the reference's `sample` [B, 263, 1, required_frames] and, as `inputs_sum`, fp64 sums of the seeded
inputs (inputs(case): the tape's x_T [n, B, 263, 1, 40] and eps [n, 3, ...], the TableBert tables), which the tests
regenerate rather than read.
"""
import importlib
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

syn = importlib.import_module("motion-diffusion-model_b200.synthetic")
OUT = os.path.join(ROOT, "tests", "golden", "dip_ar_small.npz")
L, STEPS, B, CTX, PRED, MT = 2, 3, 3, 20, 40, 7
LENGTHS, SCALES, WEIGHTS_SEED = [40, 33, 12], [7.5, 2.0, 1.0], 4
CASES = {"dyn196": dict(dynamic=True, include_prefix=True, required=196),
         "static100": dict(dynamic=False, include_prefix=False, required=100)}


def n_chunks(required):
    return required // PRED + int(required % PRED > 0)


def prompt(case, c, b):
    """The prompt of sample b in chunk c (every chunk's prompt is chunk 0's without per-chunk text)."""
    return "%s chunk %d sample %d" % (case, c if CASES[case]["dynamic"] else 0, b)


def inputs(case):
    """Seeded inputs of a case: dict(enc [n, Mt, B, C], pad [n, B, Mt], prefix, x_T [n, ...], eps [n, STEPS, ...], mask,
    lengths, scale, texts)."""
    cfg = CASES[case]
    n = n_chunks(cfg["required"])
    encs, pads, xs, eps = [], [], [], []
    for c in range(n):
        enc, pad, _ = syn.synthetic_dip_inputs(B, MT, CTX, seed=50 + (c if cfg["dynamic"] else 0))
        encs.append(enc)
        pads.append(pad)
        inp = syn.synthetic_inputs(B, nframes=PRED, steps=STEPS, seed=60 + c, lengths=LENGTHS, scale=torch.tensor(SCALES))
        xs.append(inp["tape"][0])
        eps.append(torch.stack(inp["tape"][1:]))
    _, _, prefix = syn.synthetic_dip_inputs(B, MT, CTX, seed=3)
    texts = [[prompt(case, c, b) for c in range(n)] for b in range(B)]
    return dict(enc=torch.stack(encs), pad=torch.stack(pads), prefix=prefix, x_T=torch.stack(xs), eps=torch.stack(eps),
                mask=inp["mask"], lengths=inp["lengths"], scale=inp["scale"], texts=texts)


def inputs_sum(inp):
    return np.array([float(inp[k].double().sum()) for k in ("x_T", "eps", "enc", "pad", "prefix")])


class TableBert(torch.nn.Module):
    """A BERT stand-in with the interface bert_encode_text calls (model/mdm.py:180-187): prompts -> (features
    [B, Mt, C], True where a token is present), looked up in the case's tables."""

    def __init__(self, case, enc, pad):
        super().__init__()
        self.table = {}
        for c in range(enc.shape[0]):
            for b in range(B):
                self.table[prompt(case, c, b)] = (enc[c][:, b], ~pad[c][b])

    def forward(self, texts):
        feats = torch.stack([self.table[t][0] for t in texts])
        present = torch.stack([self.table[t][1] for t in texts])
        return feats, present


def y_of(case, inp):
    """The caller's y of a case, in the reference's layout: y['text'] a list of lists with per-chunk prompts (and a
    placeholder y['text_embed'] the reference slices before encoding), else one prompt per sample."""
    cfg = CASES[case]
    n = inp["x_T"].shape[0]
    y = dict(mask=inp["mask"].clone(), lengths=inp["lengths"].clone(), scale=inp["scale"].clone(), prefix=inp["prefix"].clone())
    if cfg["dynamic"]:
        y["text"] = [list(t) for t in inp["texts"]]
        y["text_embed"] = (torch.zeros(MT, B, n, 768), torch.zeros(B, n, MT, dtype=torch.bool))
    else:
        y["text"] = [t[0] for t in inp["texts"]]
    return y


def ar_args(case):
    return SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=CASES[case]["include_prefix"])


def gen():
    from oracle import ref_harness as rh
    ns = rh.load_reference()
    args = rh.default_args(layers=L, diffusion_steps=STEPS, arch="trans_dec", text_encoder_type="bert", context_len=CTX,
                           pred_len=PRED)
    sd = syn.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=768, seed=WEIGHTS_SEED)
    out = {"meta": np.array(["DiP L=%d steps=%d B=%d ctx=%d pred=%d Mt=%d weights_seed=%d lengths=%s scales=%s; the "
                             "reference's AutoRegressiveSampler + p_sample_loop, clip_denoised=False"
                             % (L, STEPS, B, CTX, PRED, MT, WEIGHTS_SEED, LENGTHS, SCALES)])}
    for case, cfg in CASES.items():
        model, diff = rh.build(args, state_dict=sd)
        inp = inputs(case)
        model.clip_model = TableBert(case, inp["enc"], inp["pad"])
        guided = ns.sampler_util.ClassifierFreeSampleModel(model)
        tape = []
        for c in range(inp["x_T"].shape[0]):
            tape += [inp["x_T"][c]] + list(inp["eps"][c])
        sampler = ns.sampler_util.AutoRegressiveSampler(ar_args(case), diff.p_sample_loop, required_frames=cfg["required"])
        with torch.no_grad(), rh.noise_tape(tape) as proxy:
            sample = sampler.sample(guided, (B, 263, 1, cfg["required"]), clip_denoised=False, model_kwargs={"y": y_of(case, inp)})
        assert proxy._pos == len(tape), (proxy._pos, len(tape))
        out[case + "_sample"] = sample.numpy()
        out[case + "_inputs_sum"] = inputs_sum(inp)
        print(case, tuple(sample.shape))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "%.0f KB" % (os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    gen()
