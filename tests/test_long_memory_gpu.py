"""GPU: trans_dec engines with BERT text memories longer than 64 tokens (the blocked cross-attention core) against the
fp32 oracle: DiP at its released depth with Mt = 512 and guidance, a 5-chunk autoregressive DiP run with Mt = 200, and
the context_len = 0 BERT decoder at 196 frames over 50 steps with Mt = 130.  Mt = 513 is refused."""
from types import SimpleNamespace

import pytest
import torch

import b200mdm
from b200mdm._lib import B200MDMError
from conftest import default_args, rel_err

pytestmark = pytest.mark.gpu
RTOL = 1e-3


def _dec(layers, steps, seed, ctx, pred):
    args = default_args(layers=layers, diffusion_steps=steps, arch="trans_dec", text_encoder_type="bert", context_len=ctx,
                        pred_len=pred)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=layers, cond_dim=768, seed=seed)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    return b200mdm.ClassifierFreeSampleModel(model), model, diffusion, sd, args


def _gpu_tape(steps, shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g), torch.randn(steps, *shape, device="cuda", generator=g)


def test_dip_b64_mt512_guided_vs_oracle():
    """8 layers, B = 64 with guidance, Mt = 512 (ragged padding), 10 steps; the oracle follows three samples."""
    from oracle import mdm_oracle as mo, schedule_oracle as so
    B, ctx, pred, Mt, steps = 64, 20, 40, 512, 10
    cfg, model, diffusion, sd, _ = _dec(8, steps, 61, ctx, pred)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, ctx, seed=62)
    scale = torch.linspace(0.0, 7.5, B)
    lengths = torch.randint(1, pred + 1, (B,), generator=torch.Generator().manual_seed(63))
    lengths[0] = pred
    shape = (B, 263, 1, pred)
    xT, tape = _gpu_tape(steps, shape, 64)
    y = dict(mask=(torch.arange(pred)[None, None, None, :] < lengths[:, None, None, None]).cuda(), lengths=lengths.cuda(),
             text_embed=(enc.cuda(), tmask.cuda()), prefix=prefix.cuda(), scale=scale.cuda())
    out = diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape)
    assert torch.isfinite(out).all()
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    idx = [0, 37, 63]
    want = mo.sample_loop_dec(W, tabs, list(range(steps)), [xT[idx].cpu()] + [tape[k][idx].cpu() for k in range(steps)],
                              enc[:, idx], tmask[idx], prefix[idx], scale[idx], lengths[idx])
    e = rel_err(out[idx], want)
    print("DiP B=64, Mt=512, 10 steps, guidance: relative error vs oracle", e)
    assert e < RTOL


def test_dip_autoregressive_mt200_vs_oracle():
    """AutoRegressiveSampler over an 8-layer DiP engine: 5 chunks of 40 frames, Mt = 200, guidance."""
    from oracle import mdm_oracle as mo, schedule_oracle as so
    B, ctx, pred, Mt, steps, need = 2, 20, 40, 200, 3, 200
    cfg, model, diffusion, sd, args = _dec(8, steps, 71, ctx, pred)
    W = mo.OracleWeights(sd, 8)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(B, Mt, ctx, seed=72)
    scale = torch.tensor([7.5, 2.5])
    chunks = [b200mdm.synthetic_inputs(B, nframes=pred, steps=steps, seed=80 + i, scale=scale) for i in range(5)]
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    cur, buf = prefix, []
    for c in chunks:
        s = mo.sample_loop_dec(W, tabs, list(range(steps)), c["tape"], enc, tmask, cur, scale, c["lengths"])
        buf.append(s)
        cur = s[..., -ctx:]
    want = torch.cat(buf, -1)[..., :need]
    y = dict(mask=chunks[0]["mask"].cuda(), lengths=chunks[0]["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             prefix=prefix.cuda(), scale=scale.cuda())
    sampler = b200mdm.AutoRegressiveSampler(args, diffusion.p_sample_loop, required_frames=need)
    out = sampler.sample(cfg, (B, 263, 1, need), clip_denoised=False, model_kwargs={"y": y},
                         noise=torch.stack([c["tape"][0] for c in chunks]).cuda(),
                         noise_tape=torch.stack([torch.stack(c["tape"][1:]) for c in chunks]).cuda())
    e = rel_err(out, want)
    print("DiP autoregressive, 5 chunks, Mt=200: relative error vs oracle", e)
    assert e < RTOL


def test_bert_decoder_ctx0_t196_mt130_vs_oracle():
    """The context_len = 0 BERT decoder (humanml_trans_dec_512_bert-50steps): 8 layers, 196 frames, 50 steps, Mt = 130,
    guidance, ragged lengths."""
    from oracle import mdm_oracle as mo, schedule_oracle as so
    B, T, Mt, steps = 3, 196, 130, 50
    cfg, model, diffusion, sd, _ = _dec(8, steps, 91, 0, 0)
    enc, tmask, _ = b200mdm.synthetic_dip_inputs(B, Mt, 0, seed=92)
    inp = b200mdm.synthetic_inputs(B, nframes=T, steps=steps, seed=93, lengths=[196, 120, 17], scale=torch.tensor([7.5, 2.5, 1.0]))
    prefix = torch.zeros(B, 263, 1, 0)
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             scale=inp["scale"].cuda())
    out = diffusion.p_sample_loop(cfg, (B, 263, 1, T), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                  model_kwargs={"y": y}, noise_tape=torch.stack(inp["tape"][1:]).cuda())
    W = mo.OracleWeights(sd, 8)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    want = mo.sample_loop_dec(W, tabs, list(range(steps)), inp["tape"], enc, tmask, prefix, inp["scale"], inp["lengths"])
    e = rel_err(out, want)
    print("BERT decoder ctx=0, T=196, Mt=130, 50 steps: relative error vs oracle", e)
    assert e < RTOL


def test_memory_of_513_tokens_refused():
    cfg, model, diffusion, _, _ = _dec(2, 3, 4, 20, 40)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(2, 513, 20)
    x = torch.randn(2, 263, 1, 40, device="cuda")
    y = dict(mask=torch.ones(2, 1, 1, 40, dtype=torch.bool, device="cuda"), lengths=torch.tensor([40, 40]).cuda(),
             text_embed=(enc.cuda(), tmask.cuda()), prefix=prefix.cuda(), scale=torch.tensor([2.5, 1.0]).cuda())
    with pytest.raises(B200MDMError, match="512"):
        cfg(x, torch.tensor([1, 1]).cuda(), y=y)


def test_longmem_vs_reference_golden(golden):
    """The unmodified reference's DiP (Mt = 150, ragged masks, guidance) and context_len = 0 BERT decoder (T = 196,
    Mt = 100) of tests/golden/dip_longmem_small.npz: a guided forward and the DDPM loops, eager and graphed."""
    from oracle import gen_golden_longmem as gl
    g = golden("dip_longmem_small.npz")
    c = gl.DIP
    cfg, model, diffusion, _, _ = _dec(c["L"], c["steps"], c["weights_seed"], c["ctx"], c["pred"])
    inp, enc, tmask, prefix = gl.dip_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             prefix=prefix.cuda(), scale=inp["scale"].cuda())
    t = torch.full((c["B"],), 1, dtype=torch.long, device="cuda")
    assert rel_err(cfg(inp["tape"][0].cuda(), t, y=y), g["dip_fwd_cfg"]) < RTOL
    tape, xT = torch.stack(inp["tape"][1:]).cuda(), inp["tape"][0].cuda()
    for use_graph in (False, True):
        out = diffusion.p_sample_loop(cfg, (c["B"], 263, 1, c["pred"]), noise=xT, clip_denoised=False,
                                      model_kwargs={"y": y}, noise_tape=tape, use_graph=use_graph)
        assert rel_err(out, g["dip_ddpm"]) < RTOL, use_graph
    c = gl.BERT
    cfg, model, diffusion, _, _ = _dec(c["L"], c["steps"], c["weights_seed"], 0, 0)
    inp, enc, tmask = gl.bert_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=(enc.cuda(), tmask.cuda()),
             scale=inp["scale"].cuda())
    out = diffusion.p_sample_loop(cfg, (c["B"], 263, 1, c["T"]), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                  model_kwargs={"y": y}, noise_tape=torch.stack(inp["tape"][1:]).cuda())
    e = rel_err(out, g["bert_ddpm"])
    print("reference fixture: BERT decoder T=196 Mt=100 relative error", e)
    assert e < RTOL
