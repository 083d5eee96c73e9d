"""GPU: multi-prompt guidance (DESIGN.md "Multi-prompt guidance") stage by stage, and its composed step bit for bit.

The packed batch holds G = K + 1 groups of B motions (the prompts' groups, then the unconditional one).  Through
b200mdm_test_forward_taps, with the key counts and memory masks derived from y (not read from the engine):
  a. every stage of the forward over all G groups against its kernel hook (check_layer of test_forward_stages_gpu.py,
     run on the packed batch as G * B motions with halves 1): the embedding GEMM of every group, with one mutant per
     middle group that the pairing loop could miss (its rows left as the previous forward's residual); token 0; the
     conditioning rows (prompt k's text projection or action embedding of action[b, k], the unconditional group last)
     against fp64 within linear_bound, with the prompts reversed and the action packing transposed as mutants; the
     CLIP decoder's cross rows (one per group); the BERT decoder's per-group memory mask, the unconditional group
     admitting exactly the tokens some prompt admits; the G * B * T frame rows of the blend; and X0G, every group's raw
     x0, against the MODE_X0 output hook over the G * B motions;
  b. the composed output against a numpy float32 restatement over the tapped X0G, x0_u + sum_k w (x0_k - x0_u), one
     rounding per operation, k ascending; FMA-contracted, k descending, the unconditional group taken from group 0,
     the f and t strides swapped and the weight row of motion b + 1 must each differ somewhere;
  c. the step's tail, bit for bit: pred_xstart = clamp(inpaint(compose(X0G))), X0G tapped at the step's x and model
     timestep, and the sample against the update restatements of the other step tests (DDPM, DDIM eta 0 / 0.5, PLMS
     orders 1-4 and its improved-Euler step with the second forward at (mean_1, t_{i-1}), DPM-Solver++ orders 1 and 2
     with the x0 history, DDIM inversion), with and without clip_denoised, hard and soft inpainting;
  d. K = 1..5 and 8 (every middle-group pairing, the single-group tail and the maximum; K = 9 is refused), all 16
     zero / non-zero stride patterns of (b, k, f, t) and a weight stored [T, D, K, B], the four model kinds and target
     conditioning; small shapes for the sweeps and the headline shape (B = 64, T = 196, L = 8, K = 2) at one layer."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
import test_forward_stages_gpu as fs
from test_forward_stages_gpu import Record, check_layer, embed, gemm_epi, linear_bound
from test_epilogues_gpu import _step_f32, check_x_out
from test_plms_gpu import _eps, _rows, _sample
from test_reverse_gpu import _update
from oracle import dpm_oracle as do
from oracle import plms_oracle as po

pytestmark = pytest.mark.gpu
D = 512
U32 = 2.0 ** -24


# ------------------------------------------------------------------------------------------------ cases
def _actions(B, K):
    """int64 [B, K], distinct along k, so a transposed packing shows with B != K"""
    return ((7 * np.arange(B)[:, None] + np.arange(K)[None]) % 12).astype(np.int64)


def _token_prompts(B, K, Mt, g):
    """K BERT prompts of different token counts (Mt, Mt - 2, ...), each right-padded per sample, prompt 0 the most, so
    that the unconditional group's mask (where every prompt pads) is not prompt 0's"""
    pairs = []
    for k in range(K):
        n = max(2, Mt - 2 * k)
        tok = torch.randn(n, B, 768, generator=g) * 0.5
        mask = torch.zeros(B, n, dtype=torch.bool)
        for b in range(B):
            mask[b, max(1, n - (4 + b % 2 if k == 0 else (b + k) % 3)):] = True
        pairs.append((tok.cuda(), mask.cuda()))
    return pairs


def _memmask(pairs, B):
    """[G * B, Mt] uint8 (1 = padding) derived from the prompts: each prompt's mask padded to the longest, then the
    unconditional group padding where every prompt pads; and the mutant whose unconditional group takes prompt 0's"""
    Mt = max(int(t.shape[0]) for t, _ in pairs)
    m = torch.ones(len(pairs), B, Mt, dtype=torch.uint8)
    for k, (t, mk) in enumerate(pairs):
        m[k, :, :t.shape[0]] = mk.cpu().to(torch.uint8)
    unc = m.min(0).values
    return (torch.cat([m.reshape(-1, Mt), unc]).cuda().contiguous(),
            torch.cat([m.reshape(-1, Mt), m[0]]).cuda().contiguous(), Mt)


def mp_case(kind, B, T, L, K, seed, lengths=None, target=None, Mt=16, same_t=False):
    """A test_forward_stages_gpu case with K prompts set through Engine.set_cond_multi, and its packed view `p`: the
    G * B motions as a halves-1 batch, so that check_layer runs over every group unchanged."""
    c = fs.build(kind, B, T, L, seed, False, lengths=lengths, Mt=Mt, ctx=0, target=target)
    g = torch.Generator().manual_seed(seed + 5)
    G = K + 1
    c.K, c.G, c.act, c.pairs, c.embed = K, G, None, None, None
    if kind == "a2m":
        c.act = _actions(B, K)
    elif kind == "dip":                               # the BERT decoder (context_len 0)
        c.pairs = _token_prompts(B, K, Mt, g)
    else:
        c.embed = (torch.randn(K, B, 512, generator=g) * 0.5).cuda()
    w = (torch.rand(B, K, c.JF, T, generator=g) * 3 - 0.5).cuda()
    c.eng.set_cond_multi(B, T, c.y, c.pairs if kind == "dip" else c.embed, c.act, w, "cuda")
    c.w = w
    assert c.eng.groups == G and c.eng.packed_batch() == G * B
    if same_t:
        c.ts = torch.full((B,), 23, dtype=torch.long)
    p = SimpleNamespace(**vars(c))
    p.B, p.halves, p.Bp, p.M, p.scale = G * B, 1, G * B, G * B * c.S, None
    p.x = c.x.repeat(G, 1, 1, 1)
    p.kvlen = c.kvlen.repeat(G).contiguous()
    if kind == "dip":
        p.memmask, c.memmask_p0, p.Mt = _memmask(c.pairs, B)
    c.p = p
    return c


def set_weight(c, storage, strides):
    """b200mdm_set_prompt_weight straight through the C ABI (the wrapper always passes a contiguous weight); returns the
    effective w [B, K, JF, T] as numpy float32"""
    storage = storage.contiguous()
    lib = _lib.load()
    _lib.check(lib.b200mdm_set_prompt_weight(c.eng.h, c.K, ctypes.c_void_p(storage.data_ptr()), *[int(s) for s in strides],
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    c.eng._keep["prompt_weight"] = storage
    return torch.as_strided(storage, (c.B, c.K, c.JF, c.T), strides).cpu().numpy().astype(np.float32)


def weight_pattern(c, bits, g):
    """(storage, strides) of the stride pattern `bits` over (b, k, f, t): a dimension whose bit is clear has stride 0"""
    full = (c.B, c.K, c.JF, c.T)
    size = [n if bits >> (3 - i) & 1 else 1 for i, n in enumerate(full)]
    s = torch.rand(*size, generator=g) * 3 - 0.5
    st = list(torch.empty(*size).stride())
    strides = [st[i] if size[i] > 1 else 0 for i in range(4)]
    return s.cuda(), strides


# ------------------------------------------------------------------------------------------------ b: the composition
def compose32(x0g, w, K, order=None, fma=False, uncond=None):
    """x0_u + sum_k w[:, k] (x0_k - x0_u) in numpy float32, one rounding per operation; x0g [G * B, JF, T]"""
    B = w.shape[0]
    xg = x0g.reshape(K + 1, B, *x0g.shape[1:])
    xu = xg[K if uncond is None else uncond]
    x = xu.copy()
    for k in (order if order is not None else range(K)):
        wk = w[:, k]
        d = xg[k] - xu
        x = do.fma32(wk, d, x) if fma else (x + wk * d).astype(np.float32)
    return x


def _differ(a, b):
    return int((np.ascontiguousarray(a).view(np.int32) != np.ascontiguousarray(b).view(np.int32)).sum())


def check_compose(rec, name, out, x0g, w, K, mutants=True):
    """the composed output bit for bit against compose32 over the tapped X0G, and the mutants that apply"""
    B = w.shape[0]
    got, xg = out.reshape(B, *x0g.shape[1:]).cpu().numpy(), x0g.cpu().numpy()
    n = _differ(got, compose32(xg, w, K))
    print("  %-44s %d differing elements" % (name + ": composition", n))
    if n:
        rec.bad.append("%s: the composition differs from its float32 restatement in %d elements" % (name, n))
    if not mutants:
        return
    muts = {"FMA-contracted": compose32(xg, w, K, fma=True), "unconditional group from group 0": compose32(xg, w, K, uncond=0)}
    if K > 1:
        muts["k descending"] = compose32(xg, w, K, order=range(K - 1, -1, -1))
    if B > 1 and (w != np.roll(w, -1, 0)).any():
        muts["weight row of motion b + 1"] = compose32(xg, np.roll(w, -1, 0), K)
    for mname, m in muts.items():
        nm = _differ(got, m)
        print("    mutant %-37s %d differing elements" % (mname, nm))
        if nm == 0:
            rec.bad.append("%s: mutant %s is indistinguishable" % (name, mname))


# ------------------------------------------------------------------------------------------------ a: the stages
def check_entry_mp(c, t, l, prev_ln3, rec):
    """embedding (all groups, a missed middle group as mutant), token 0, conditioning rows, cross rows / memory"""
    p, B, G, K, S, d = c.p, c.B, c.G, c.K, c.S, D
    w_in, b_in = c.W["input_process.poseEmbedding.weight"], c.W["input_process.poseEmbedding.bias"]
    ref = embed(p.x.reshape(G * B, c.JF, c.T).contiguous(), w_in, b_in, c.pe, c.s_off, 1)
    rec.same("embedding GEMM, %d groups" % G, t["EMBED"], ref)
    for grp in range(1, G - 1):      # the groups the pairing loop launches: left as the previous forward's residual
        mut = ref.clone().view(G, B * S, 2 * d)
        mut[grp] = prev_ln3.view(G, B * S, 2 * d)[grp]
        rec.teeth("embedding: group %d missed by the pairing" % grp, t["EMBED"], mut.view(-1, 2 * d))
    te = t["TEMB"] + (c.g if c.g is not None else 0)
    if c.dip:
        rec.same("token rows untouched by the memory build", t["TOK0"], t["EMBED"])
        check_memory(c, t, rec)
    else:
        hs, es = t["TOK0"].view(G * B, S, 2 * d), t["EMBED"].view(G * B, S, 2 * d)
        rec.same("frame rows untouched by token 0", hs[:, 1:], es[:, 1:])
        ter = te.repeat(G, 1)
        v = ter + c.pe[0] if c.dec else (t["CONDPROJ"] + ter) + c.pe[0]
        hi = v.half()
        rec.same("token-0 rows, %d groups" % G, hs[:, 0], torch.cat([hi, (v - hi.float()).half()], -1))
        check_condproj(c, t, rec)
    if c.dec and not c.dip:
        rows = c.eng.test_cross_rows(int(c.ts[0]), device="cuda")
        assert torch.equal(c.eng.test_cross_rows(int(c.ts[0]), G, "cuda"), rows)
        with pytest.raises(ValueError):
            c.eng.test_cross_rows(int(c.ts[0]), 2 if G != 2 else 1, "cuda")     # the CFG rows of the batch
        rec.same("cross rows [L, G*B, d] = b200mdm_test_cross_rows", t["CROSS_C"], rows)
        rec.teeth("cross rows: groups rotated", t["CROSS_C"], rows.view(c.L, G, B, d).roll(1, 1).reshape(c.L, G * B, d))
    if l == 0:
        rec.same("layer-0 entry", t["L_IN"], t["TOK0"])


def check_condproj(c, t, rec):
    B, K, d = c.B, c.K, D
    cp = t["CONDPROJ"]
    if c.act is not None:
        emb = c.W["embed_action.action_embedding"]
        packed = torch.from_numpy(c.act.T.reshape(-1).copy()).cuda()     # a[k * B + b] = action[b, k]
        rec.same("action rows, group-major", cp[:K * B], emb[packed])
        rec.teeth("action rows: packing transposed", cp[:K * B], emb[torch.from_numpy(c.act.reshape(-1).copy()).cuda()])
        rec.same("unconditional action rows = 0", cp[K * B:], torch.zeros(B, d, device="cuda"))
        return
    te = c.embed.reshape(K * B, -1).double()
    w, b = c.W["embed_text.weight"].double(), c.W["embed_text.bias"].double()
    want = te @ w.t() + b
    got = cp[:K * B].double()
    muts = {"bias dropped": (got - want + b).abs()}
    if K > 1:
        muts["prompts reversed"] = (got - (c.embed.flip(0).reshape(K * B, -1).double() @ w.t() + b)).abs()
    rec.bound("text rows of %d prompts (fp64)" % K, (got - want).abs(), linear_bound(te, w, b), muts)
    rec.same("unconditional rows = embed_text.bias", cp[K * B:], c.W["embed_text.bias"].expand(B, d))


def check_memory(c, t, rec):
    """the BERT decoder's memory rows against fp64, the all-layer K/V GEMM against its hook, and the per-group mask"""
    B, K, G, d, Mt = c.B, c.K, c.G, D, c.p.Mt
    w, b = c.W["embed_text.weight"].double(), c.W["embed_text.bias"].double()
    tok = torch.zeros(K, B, Mt, 768, dtype=torch.float64, device="cuda")
    for k, (tk, _) in enumerate(c.pairs):
        tok[k, :, :tk.shape[0]] = tk.permute(1, 0, 2).double()
    proj = torch.cat([(tok @ w.t() + b).reshape(K * B, Mt, d), b.expand(B, Mt, d)])
    pbound = torch.cat([linear_bound(tok, w, b).reshape(K * B, Mt, d), torch.zeros(B, Mt, d, dtype=torch.float64, device="cuda")])
    ref, tbound, _ = fs.temb64(c, c.ts.cuda())
    want = proj + ref.repeat(G, 1)[:, None]
    m = t["MEM16"].view(G * B, Mt, 2 * d)
    got = m[..., :d].double() + m[..., d:].double()
    bnd = pbound + tbound.repeat(G, 1)[:, None] + U32 * want.abs() + 2.0 ** -22 * want.abs() + 2.0 ** -25
    muts = {"text bias dropped": (got - want + b).abs()}
    if K > 1:
        rev = torch.cat([proj[:K * B].view(K, B, Mt, d).flip(0).reshape(K * B, Mt, d), proj[K * B:]])
        muts["prompts reversed"] = (got - rev - ref.repeat(G, 1)[:, None]).abs()
    rec.bound("memory rows of %d prompts + temb (fp64)" % K, (got - want).abs(), bnd, muts)
    wkv = torch.cat([fs.lw(c, l, "multihead_attn.in_proj_weight")[d:] for l in range(c.L)])
    bkv = torch.cat([fs.lw(c, l, "multihead_attn.in_proj_bias")[d:] for l in range(c.L)])
    rec.same("all-layer K/V GEMM, %d groups" % G, t["KVC16"], gemm_epi(t["MEM16"][:, :d].contiguous(), fs.f16(wkv), bkv, 1))


def check_masks(c, t, l, rec):
    """the BERT decoder's cross-attention core with the prompts' masks rotated (K >= 2) must give other bits; the
    unconditional group with prompt 0's mask is printed only: its tokens are all equal, so every mask that admits one of
    them gives the same bits (pack_text_mask in engine.cu)"""
    if not c.dip or c.K < 2:
        return
    p, d, B, K = c.p, D, c.B, c.K
    ld = c.L * 2 * d
    xat = t["L_XATT"][:, :d]
    rot = p.memmask.clone()
    rot[:K * B] = p.memmask[:K * B].view(K, B, -1).roll(1, 0).reshape(K * B, -1)
    rec.teeth("L%d cross core: prompt masks rotated" % l, xat,
              fs.cross_attention(t["L_QC"], t["KVC16"], l * 2 * d, ld, rot.contiguous(), p.Bp, c.S, p.Mt))
    assert not torch.equal(c.memmask_p0, p.memmask)
    mut = fs.cross_attention(t["L_QC"], t["KVC16"], l * 2 * d, ld, c.memmask_p0, p.Bp, c.S, p.Mt)
    n = int((mut.contiguous().view(torch.int16) != xat.contiguous().view(torch.int16)).sum())
    print("    (unconditional group with prompt 0's mask: %d differing elements, equal tokens)" % n)


def run_stages(c, title, layers=None, weights=True):
    """a (every stage at `layers`, default the first and last) and b (the composition, and with `weights` every stride
    pattern and a weight stored [T, D, K, B]) for case c"""
    rec = Record(title)
    plain = c.eng.denoise(c.x, c.ts)
    layers = layers if layers is not None else sorted({c.L - 1, 0}, reverse=True)
    _, last = c.eng.forward_taps(c.x, c.ts, c.L - 1, names=["L_LN3"])     # the residual a missed group would keep
    torch.cuda.synchronize()
    w = c.w.cpu().numpy()
    for l in layers:
        out, t = c.eng.forward_taps(c.x, c.ts, l)
        torch.cuda.synchronize()
        check_entry_mp(c, t, l, last["L_LN3"], rec)
        check_layer(c.p, l, t, t["X0G"], rec)      # (the output stage: X0G, every group's raw x0)
        check_masks(c, t, l, rec)
        rec.same("tapped forward = b200mdm_denoise", out, plain)
        check_compose(rec, "L%d forward" % l, out, t["X0G"], w, c.K)
    if weights:
        g = torch.Generator().manual_seed(99)
        x0g = t["X0G"]
        for bits in range(16):
            storage, strides = weight_pattern(c, bits, g)
            we = set_weight(c, storage, strides)
            out = c.eng.denoise(c.x, c.ts)
            check_compose(rec, "strides (b k f t) %s" % format(bits, "04b"), out, x0g, we, c.K, mutants=bits == 15)
            if bits == 15 and c.T <= c.JF:     # the kernel reading f with t's stride and t with f's (inside the storage)
                sw = torch.as_strided(storage, (c.B, c.K, c.JF, c.T), (strides[0], strides[1], strides[3], strides[2]))
                n = _differ(out.reshape(c.B, c.JF, c.T).cpu().numpy(), compose32(x0g.cpu().numpy(), sw.cpu().numpy(), c.K))
                print("    mutant %-37s %d differing elements" % ("f and t strides swapped", n))
                if n == 0:
                    rec.bad.append("mutant f and t strides swapped is indistinguishable")
        # a non-contiguous weight, stored [T, D, K, B]: strides 1, B, K B, D K B
        st = (torch.rand(c.T, c.JF, c.K, c.B, generator=g) * 3 - 0.5).cuda()
        we = set_weight(c, st, (1, c.B, c.K * c.B, c.JF * c.K * c.B))
        check_compose(rec, "weight stored [T, D, K, B]", c.eng.denoise(c.x, c.ts), x0g, we, c.K)
        c.eng.set_cond_multi(c.B, c.T, c.y, c.pairs if c.dip else c.embed, c.act, c.w, "cuda")
    rec.done()


# ------------------------------------------------------------------------------------------------ a, b, d: the sweeps
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 8])
def test_stages_trans_enc_text(K):
    c = mp_case("enc", 3, 24, 2, K, 300 + K, lengths=[24, 1, 11])
    run_stages(c, "trans_enc text, K=%d (G=%d), B=3 T=24 L=2" % (K, K + 1))


@pytest.mark.parametrize("K", [2, 5])
def test_stages_action_model(K):
    c = mp_case("a2m", 3, 40, 2, K, 320 + K, lengths=[40, 1, 23])
    assert c.JF == 150
    run_stages(c, "a2m (150 features), K=%d, B=3 T=40 L=2" % K, weights=K == 5)


@pytest.mark.parametrize("K", [1, 4])
def test_stages_clip_decoder(K):
    c = mp_case("dec_emb", 3, 24, 2, K, 340 + K, lengths=[24, 1, 9], same_t=True)
    run_stages(c, "CLIP decoder, K=%d, B=3 T=24 L=2" % K, weights=K == 4)


@pytest.mark.parametrize("K", [1, 3])
def test_stages_bert_decoder(K):
    c = mp_case("dip", 3, 40, 2, K, 360 + K, lengths=[40, 1, 17], Mt=12)
    assert c.p.Mt == 12 and (c.p.memmask[-3:].cpu() <= c.p.memmask[:3].cpu()).all()
    run_stages(c, "BERT decoder ctx 0, K=%d, Mt=12..%d, B=3 T=40 L=2" % (K, 12 - 2 * (K - 1)), weights=K == 3)


def test_stages_target_conditioning():
    c = mp_case("enc", 3, 24, 2, 2, 380, lengths=[24, 1, 11], target="single")
    run_stages(c, "trans_enc text + target, K=2, B=3 T=24 L=2", weights=False)


def test_stages_headline_shape():
    """B = 64, T = 196, L = 8, K = 2: the stages at the last layer and the composition"""
    c = mp_case("enc", 64, 196, 8, 2, 390, lengths=fs._lengths(64, 196, 3))
    run_stages(c, "trans_enc text, K=2, B=64 T=196 L=8", layers=[7], weights=False)


def test_nine_prompts_are_refused():
    c = fs.build("enc", 2, 16, 1, 399, False)
    mp = b200mdm.MultiPromptSampleModel(c.model)
    y = dict(prompt_embed=torch.zeros(9, 2, 512), prompt_weight=torch.ones(2, 9, 1, 1))
    with pytest.raises(ValueError, match="1 .. 8"):
        mp.prompts(y, (2, 263, 1, 16))
    with pytest.raises(_lib.B200MDMError) as ei:
        c.eng.set_cond_multi(2, 16, {}, torch.zeros(9, 2, 512), None, torch.ones(2, 9, 1, 1), "cuda")
    assert ei.value.code == _lib.EINVAL


# ------------------------------------------------------------------------------------------------ c: the step's tail
def _tail_case(kind, K, seed):
    c = mp_case(kind, 3, 24, 2, K, seed, lengths=[24, 1, 11])
    c.mp = b200mdm.MultiPromptSampleModel(c.model)
    g = torch.Generator().manual_seed(seed + 9)
    c.imask = torch.rand(c.shape, generator=g) < 0.3
    c.motion = torch.rand(c.shape, generator=g) * 2.4 - 1.2
    c.soft = torch.rand(c.shape, generator=g)
    c.soft[..., :3] = 1.0
    c.soft[..., -3:] = 0.0
    return c


def _y(c, inpaint):
    y = dict(mask=c.y["mask"], lengths=c.y["lengths"], prompt_weight=c.w)
    y["prompt_embed"] = c.embed
    if inpaint == "hard":
        y.update(inpainting_mask=c.imask.cuda(), inpainted_motion=c.motion.cuda())
    elif inpaint == "soft":
        y.update(inpainting_weight=c.soft.cuda(), inpainted_motion=c.motion.cuda())
    return y


def _pred(c, x, t_model, clip, inpaint):
    """clamp(inpaint(compose(X0G))) with X0G tapped at (x, model timestep t_model), torch fp32 on the CPU"""
    out, taps = c.eng.forward_taps(x, torch.full((c.B,), int(t_model), dtype=torch.long), 0, names=["X0G"])
    x0 = torch.from_numpy(compose32(taps["X0G"].cpu().numpy(), c.w.cpu().numpy(), c.K)).reshape(c.shape)
    assert torch.equal(out.cpu(), x0)
    if inpaint == "hard":
        x0 = torch.where(c.imask, c.motion, x0)
    elif inpaint == "soft":
        a, b = (1 - c.soft) * x0, c.soft * c.motion
        x0 = torch.where(c.soft >= 1, c.motion, torch.where(c.soft <= 0, x0, a + b))
    return x0.clamp(-1, 1) if clip else x0


TAILS = [(False, None), (True, None), (False, "hard"), (True, "hard"), (False, "soft")]


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("kind", ["enc", "dec_emb"])
def test_tail_ddpm_ddim(kind):
    c = _tail_case(kind, 3, 400)
    d, tm = c.diffusion, c.diffusion.timestep_map
    g = torch.Generator().manual_seed(1)
    x = torch.randn(c.shape, generator=g).cuda()
    noise = torch.randn(c.shape, generator=g)
    for i in (0, 17, d.num_timesteps - 1):
        t = torch.full((c.B,), i, dtype=torch.long, device="cuda")
        for clip, inp in TAILS:
            for name, fn, mode, eta in (("ddpm", d.p_sample, _lib.MODE_DDPM, 0.0), ("ddim0", d.ddim_sample, _lib.MODE_DDIM, 0.0),
                                        ("ddim0.5", d.ddim_sample, _lib.MODE_DDIM, 0.5)):
                kw = {} if name == "ddpm" else {"eta": eta}
                out = fn(c.mp, x, t, clip_denoised=clip, model_kwargs={"y": _y(c, inp)}, noise=noise.cuda(), **kw)
                pred = _pred(c, x, tm[i], clip, inp)
                ok = _bits(out["pred_xstart"].cpu(), pred)
                print("%s %s i %d clip %d inpaint %s: pred_xstart == clamp(inpaint(compose(X0G))) %s"
                      % (kind, name, i, clip, inp, ok))
                assert ok
                row = d.schedule_rows(eta)[i]
                if i != 0:
                    check_x_out(mode, pred, x.cpu(), noise, out["sample"], row=row)
                else:
                    want = _step_f32(mode, pred.numpy(), x.cpu().numpy(), noise.numpy(), row)
                    assert _differ(out["sample"].cpu().numpy(), want) == 0
    # DDPM with the engine's Philox noise: the same step with the noise its stream draws
    _philox_step(c, x)


def _philox_step(c, x):
    """one DDPM step of a loop drawing its noise from the engine's Philox stream (b200mdm_sample_loop_range)"""
    d, eng, i = c.diffusion, c.eng, 17
    t = torch.full((c.B,), i, dtype=torch.long, device="cuda")
    d.p_sample(c.mp, x, t, clip_denoised=False, model_kwargs={"y": _y(c, None)}, noise=torch.zeros(c.shape, device="cuda"))
    eng.set_noise_stream(5, 0)
    out = torch.empty_like(x)
    eng.sample_loop_range(_lib.MODE_DDPM, i, 1, x, out, None, 0, False)
    pred = _pred(c, x, d.timestep_map[i], False, None)
    nz = eng.philox_normal(c.shape, 5, 0, i, "cuda").cpu()
    want = _step_f32(_lib.MODE_DDPM, pred.numpy(), x.cpu().numpy(), nz.numpy(), d.schedule_rows(0.0)[i])
    n = _differ(out.cpu().numpy(), want)
    print("DDPM step i %d with Philox noise: %d differing elements" % (i, n))
    assert n == 0


def test_tail_plms():
    c = _tail_case("enc", 3, 410)
    d, tm = c.diffusion, c.diffusion.timestep_map
    g = torch.Generator().manual_seed(2)
    x = torch.randn(c.shape, generator=g).cuda()
    hist = [torch.randn(c.shape, generator=g) for _ in range(3)]
    i = 9
    t = torch.full((c.B,), i, dtype=torch.long, device="cuda")
    xc = x.cpu()
    for clip, inp in TAILS:
        for order, n_old in ((1, 0), (2, 1), (3, 2), (4, 3)):
            out = d.plms_sample(c.mp, x, t, clip_denoised=clip, model_kwargs={"y": _y(c, inp)}, order=order,
                                old_out={"old_eps": [h.cuda() for h in hist[:n_old]]})
            x0 = _pred(c, x, tm[i], clip, inp)
            assert _bits(out["pred_xstart"].cpu(), x0), (order, clip, inp)
            ep = po.ab_combine([h.clone() for h in hist[:n_old]] + [_eps(d, xc, i, x0)], order)
            ok = torch.equal(out["sample"].cpu(), _sample(d, xc, i, ep, x0))
            print("PLMS order %d clip %d inpaint %s: sample bit-exact %s" % (order, clip, inp, ok))
            assert ok
    for i in (9, 0):                  # the improved-Euler step; its second forward at i - 1 (i = 0: the last index)
        t = torch.full((c.B,), i, dtype=torch.long, device="cuda")
        for clip in (False, True):
            out = d.plms_sample(c.mp, x, t, clip_denoised=clip, model_kwargs={"y": _y(c, None)}, order=2)
            x0 = _pred(c, x, tm[i], clip, None)
            assert _bits(out["pred_xstart"].cpu(), x0)
            eps0 = _eps(d, xc, i, x0)
            _, _, sq, s1 = _rows(d, i)
            mean1 = x0 * sq + s1 * eps0
            j = i - 1 if i > 0 else d.num_timesteps - 1
            x0b = _pred(c, mean1.cuda(), tm[j], clip, None)
            ep = (eps0 + _eps(d, mean1, j, x0b)) / 2
            ok = torch.equal(out["sample"].cpu(), _sample(d, xc, i, ep, x0))
            print("PLMS improved Euler i %d clip %d: sample bit-exact %s" % (i, clip, ok))
            assert ok


@pytest.mark.parametrize("order", [1, 2])
def test_tail_dpm_solver(order):
    c = _tail_case("enc", 3, 420 + order)
    d = c.diffusion
    n = d.num_timesteps
    rows = d.schedule_dpm_rows()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(c.shape, generator=g).cuda()
    for clip, inp in TAILS:
        it = d.dpm_solver_sample_loop_progressive(c.mp, c.shape, noise=x, clip_denoised=clip, model_kwargs={"y": _y(c, inp)},
                                                  order=order)
        xin, prev = x.cpu(), None
        for k, step in enumerate(it):           # every step of the loop, indices n - 1 .. 0
            i = n - 1 - k
            x0 = _pred(c, xin.cuda(), d.timestep_map[i], clip, inp)
            assert _bits(step["pred_xstart"].cpu(), x0), (i, clip, inp)
            second = order == 2 and k > 0 and i > 0
            want = do.update32(rows[i], xin.numpy(), x0.numpy(), prev.numpy() if second else None)
            nd = _differ(step["sample"].cpu().numpy(), want)
            if nd or i in (n - 1, n - 2, 0):
                print("DPM-Solver++ order %d i %d clip %d inpaint %s: %d differing elements" % (order, i, clip, inp, nd))
            assert nd == 0
            xin, prev = step["sample"].cpu(), x0


def test_tail_ddim_inversion():
    c = _tail_case("enc", 3, 430)
    d = c.diffusion
    g = torch.Generator().manual_seed(4)
    x = torch.randn(c.shape, generator=g).cuda()
    for i in (0, 17, d.num_timesteps - 1):
        t = torch.full((c.B,), i, dtype=torch.long, device="cuda")
        for clip, inp in TAILS:
            out = d.ddim_reverse_sample(c.mp, x, t, clip_denoised=clip, model_kwargs={"y": _y(c, inp)})
            x0 = _pred(c, x, d.timestep_map[i], clip, inp)
            assert _bits(out["pred_xstart"].cpu(), x0), (i, clip, inp)
            ok = torch.equal(out["sample"].cpu(), _update(d, x.cpu(), i, x0))
            print("DDIM inversion i %d clip %d inpaint %s: sample bit-exact %s" % (i, clip, inp, ok))
            assert ok
