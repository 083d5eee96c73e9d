"""GPU: the engine at every feature width JF = njoints * nfeats it accepts.  The width sets the tail geometry of the
hand-written kernels: the zero pad columns of the input projection (Kp = ceil8(JF)), the embedding GEMM's K tail
(3 Kp mod 64), the output GEMM's N (ceil96(JF)) and, in its epilogue, the last live 32-column chunk and the dead chunks
past it, and the variational bound's chunk count ceil(JF / 32).

  * every kernel hook at JF in WIDTHS (K below one k-block, exact chunks and tiles, tiles with one live column, N = 384):
    b200mdm_test_embed against fp64 (the bounds of test_epilogues_gpu.py), b200mdm_test_out_step (modes 0 / 1 / 2,
    clamp, bool inpainting) against fp64 and its x_out bit for bit, b200mdm_test_out_dpm (orders 1 and 2) and
    b200mdm_test_out_vb bit for bit against their fp32 restatements, the reduced bound terms against the fp64 mean over
    exactly JF * T elements, and b200mdm_test_out_weight (every update family; fractional, 0 and 1 weights) bit for bit.
    Every output lies inside guard bands of a sentinel bit pattern at least one [JF, T] sample wide, and exactly the
    elements of the output are written; the per-sample inputs (x, x_t, x_start, noise, motion, weights) and the weights
    and output bias are followed by NaN (the inpainting mask by ones, which select the motion's NaN), so a read past the
    last sample's last column shows.  Width-specific mutants, evaluated on the host, must miss their bounds by
    MUTANT_MARGIN;
  * the engine at KIT's 251 features: every forward and loop of tests/golden/kit_small.npz (the unmodified reference)
    within 1e-3 relative, graph and eager runs bit-identical; UESTC's 40 actions; DPM-Solver++, DDIM inversion, a
    HandshakeSampleModel DDIM loop, a soft-weighted DDIM loop and DiP's autoregressive chain (each chunk's prefix handed
    over on the device) against their fp32 oracles; the headline shape (B = 64, T = 196, L = 8, guidance 2.5, 50 DDIM
    steps) on 3 samples.  DiP's forward stages and a 3-step DiP loop at 251: tests/test_forward_stages_gpu.py.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.diffusion import gaussian_diffusion as gd
from b200mdm.diffusion import respace as rs
from conftest import default_args, rel_err
from oracle import dec_emb_oracle as deo
from oracle import double_take_oracle as dt
from oracle import dpm_oracle as do
from oracle import gen_golden_kit as gk
from oracle import handshake_oracle as ho
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import reverse_oracle as ro
from oracle import schedule_oracle as so
from oracle import vb_oracle as vo
from precision_cases import rel_err_per_sample
from test_ar_chain_gpu import build as build_chain, chain_against_fp32_oracle
from test_double_take_gpu import FAMILIES
from test_epilogues_gpu import CLIP, SCHED_ROW, U32, check, check_x_out, embed_reference, out_reference, split16
from test_vb_gpu import T0_ABS_BITS, _restate, _t0_bound

pytestmark = pytest.mark.gpu
WIDTHS = [1, 32, 96, 97, 150, 251, 263, 289]
D = 512
RTOL = 1e-3
GUARD = 4096
SENT32 = 0x7FC5A5A5     # quiet-NaN bit patterns no kernel writes
SENT16 = 0x7E5A


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def geometry(JF):
    """(Kp, pad columns, N_out, chunks, last chunk's first column)."""
    Kp = (JF + 7) // 8 * 8
    nc = (JF + 31) // 32
    return Kp, Kp - JF, (JF + 95) // 96 * 96, nc, 32 * (nc - 1)


class Guarded:
    """An output of n elements inside sentinel guard bands of max(GUARD, `sample`) elements on each side."""

    def __init__(self, shape, dtype=torch.float32, sample=0):
        self.n = int(np.prod(shape))
        self.g = max(GUARD, sample)
        self.sent = SENT32 if dtype == torch.float32 else SENT16
        bits = torch.int32 if dtype == torch.float32 else torch.int16
        self.buf = torch.full((2 * self.g + self.n,), self.sent, dtype=bits, device="cuda")
        self.t = self.buf[self.g:self.g + self.n].view(dtype).view(shape)

    def check(self, name, live=None):
        """Exactly the elements of `live` (a bool mask over the output; default all of it) were written."""
        w = self.buf != self.sent
        inside = w[self.g:self.g + self.n]
        want = torch.ones_like(inside) if live is None else live.reshape(-1)
        outside = int(w[:self.g].sum() + w[self.g + self.n:].sum())
        print("  guard %s: %d of %d written where expected, %d elsewhere, %d outside the output" % (
            name, int((inside & want).sum()), int(want.sum()), int((inside & ~want).sum()), outside))
        assert outside == 0, "%s: writes in the guard bands" % name
        assert torch.equal(inside, want), "%s: written elements differ from the output's" % name


def nan_tail(t, extra):
    """A copy of t followed by `extra` NaN elements (the buffer a read past t's end would reach)."""
    buf = torch.full((t.numel() + extra,), float("nan"), dtype=t.dtype, device="cuda")
    buf[:t.numel()] = t.reshape(-1)
    return buf[:t.numel()].view(t.shape)


def _inputs(g, B, JF, T, halves, s_off):
    """The output hooks' inputs: hres [hi | lo] of a random residual stream, scale, W_out, b_out, x_t; the per-sample
    inputs and W_out / b_out are followed by a NaN sample."""
    S = T + s_off
    h = torch.randn(halves * B * S, D, device="cuda", generator=g) * 1.2
    hh, hl = split16(h)
    hres = torch.cat([hh, hl], 1).contiguous()
    scale = torch.tensor([[0.0, 1.0, 2.5, 7.5][i % 4] for i in range(B)], device="cuda") if halves == 2 else None
    w = nan_tail(torch.randn(JF, D, device="cuda", generator=g) / D ** 0.5, D)
    b = nan_tail(torch.randn(JF, device="cuda", generator=g) * 0.1, 96)
    xt = nan_tail(torch.randn(B, JF, T, device="cuda", generator=g), JF * T)
    return hh, hl, hres, scale, w, b, xt


def _x0(lib, hres, scale, w, b, xt, flags, mask, motion, s_off, halves):
    B, JF, T = xt.shape
    out, pred = Guarded((B, JF, T), sample=JF * T), Guarded((B, JF, T), sample=JF * T)
    _lib.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w), _p(b), _p(xt), None, None, _lib.MODE_X0, flags,
                                         _p(mask), _p(motion), _p(out.t), _p(pred.t), B, JF, T, D, s_off, halves, _stream()))
    torch.cuda.synchronize()
    out.check("x0 hook x_out JF=%d" % JF)
    pred.check("x0 hook pred_xstart JF=%d" % JF)
    return pred.t


# ------------------------------------------------------------------------------------------------ embedding
@pytest.mark.parametrize("JF", WIDTHS)
def test_embed_width(JF):
    """pack_input -> split_weight -> EpiEmbed at width JF: encoder rows with and without the CFG copy, and DiP's 20
    prefix rows; the residual stream against fp64, written exactly."""
    L, lib = _lib, _lib.load()
    Kp, pad, _, _, _ = geometry(JF)
    print("JF=%d: Kp=%d (%d pad columns), embedding K = %d = %d x 64 + %d" % (JF, Kp, pad, 3 * Kp, 3 * Kp // 64, 3 * Kp % 64))
    for B, T, s_off, halves in ((3, 40, 1, 2), (3, 24, 1, 1), (2, 24, 20, 2)):
        S = T + s_off
        g = torch.Generator(device="cuda").manual_seed(JF * 10 + s_off + halves)
        x = nan_tail(torch.randn(B, JF, T, device="cuda", generator=g), JF * T)
        w = nan_tail(torch.randn(D, JF, device="cuda", generator=g) / JF ** 0.5, JF)
        b = torch.randn(D, device="cuda", generator=g) * 0.1
        pe = torch.randn(S + 3, D, device="cuda", generator=g) * 0.5
        MB = B * S
        hres = Guarded((halves * MB, 2 * D), torch.float16, sample=S * 2 * D)
        L.check(lib.b200mdm_test_embed(_p(x), _p(w), _p(b), _p(pe), _p(hres.t), B, JF, T, D, s_off, halves, _stream()))
        torch.cuda.synchronize()
        hres.check("embed JF=%d" % JF)
        out = hres.t
        if halves == 2:
            assert torch.equal(out[:MB].view(torch.int16), out[MB:].view(torch.int16)), "CFG copies differ"
        got = out[:MB, :D].double() + out[:MB, D:].double()
        ref, bound, mutants = embed_reference(x, w, b, pe, s_off)
        if pad:
            # the split run past JF: the pad columns of both operands hold the last live column's values
            xr = torch.zeros(B, S, JF, device="cuda")
            xr[:, s_off:] = x.transpose(1, 2)
            xr = xr.view(MB, JF)
            bpe = (b.double() + pe.double()[:S])[torch.arange(MB, device="cuda") % S]

            def rep(t):
                return torch.cat([t.double(), t[:, -1:].double().expand(-1, pad)], 1)
            xh, xl = split16(xr)
            wh, wl = split16(w)
            p3 = torch.cat([rep(xh), rep(xl), rep(xh)], 1) @ torch.cat([rep(wh), rep(wh), rep(wl)], 1).t() + bpe
            mutants["pad columns hold column JF - 1"] = (p3 - ref).abs()
        check("embed JF=%d B=%d T=%d s_off=%d halves=%d" % (JF, B, T, s_off, halves), (got - ref).abs(), bound, mutants)


# ------------------------------------------------------------------------------------------------ output step
@pytest.mark.parametrize("JF", WIDTHS)
def test_out_step_width(JF):
    """EpiOut<OutStep> at width JF, modes 0 / 1 / 2 with the clamp and bool inpainting: pred_xstart against the fp64
    bound, x_out bit for bit; both written exactly."""
    lib = _lib.load()
    _, _, N, nc, c0 = geometry(JF)
    print("JF=%d: N_out=%d, %d chunks, last live chunk [%d, %d) with %d live columns, %d dead columns" % (
        JF, N, nc, c0, c0 + 32, JF - c0, N - JF))
    B, T, s_off = 4, 40, 1
    for mode, halves, flags, inpaint in ((0, 1, 0, False), (1, 2, CLIP, True), (2, 2, 0, False), (2, 2, CLIP, True)):
        g = torch.Generator(device="cuda").manual_seed(JF * 10 + mode + flags)
        hh, hl, hres, scale, w, b, xt = _inputs(g, B, JF, T, halves, s_off)
        noise = nan_tail(torch.randn(B, JF, T, device="cuda", generator=g), JF * T)
        row = torch.tensor(SCHED_ROW, device="cuda")
        mask = (torch.rand(B, JF, T, device="cuda", generator=g) < 0.3) if inpaint else None
        mask8 = None
        if inpaint:   # followed by a sample of ones: a read past the end takes the motion's NaN tail
            buf = torch.ones(B * JF * T + JF * T, dtype=torch.uint8, device="cuda")
            buf[:B * JF * T] = mask.reshape(-1)
            mask8 = buf[:B * JF * T].view(B, JF, T)
        motion = nan_tail(torch.rand(B, JF, T, device="cuda", generator=g) * 1.8 - 0.9, JF * T) if inpaint else None
        xout, pred = Guarded((B, JF, T), sample=JF * T), Guarded((B, JF, T), sample=JF * T)
        _lib.check(lib.b200mdm_test_out_step(_p(hres), _p(scale), _p(w), _p(b), _p(xt), _p(noise), _p(row), mode, flags,
                                             _p(mask8), _p(motion), _p(xout.t), _p(pred.t), B, JF, T, D, s_off, halves,
                                             _stream()))
        torch.cuda.synchronize()
        xout.check("x_out JF=%d mode=%d" % (JF, mode))
        pred.check("pred_xstart JF=%d mode=%d" % (JF, mode))
        ref, bound, v_swapped, vl, wh = out_reference(hh, hl, scale, w, b, B, T, s_off, halves)

        def post(t):
            t = t.view(B, T, JF).permute(0, 2, 1)
            if inpaint:
                t = torch.where(mask, motion.double(), t)
            return t.clamp(-1, 1) if flags & CLIP else t
        ref_p = post(ref)
        mutants = {"A_lo W_hi dropped": (post(ref - vl @ wh.t()) - ref_p).abs()}
        if halves == 2:
            mutants["scale applied to the uncond half"] = (post(v_swapped @ w.double().t() + b.double()) - ref_p).abs()
        if JF - c0 >= 2:
            shifted = ref_p.clone()
            shifted[:, c0:JF - 1] = ref_p[:, c0 + 1:JF]
            mutants["last live chunk: column j read from j + 1"] = (shifted - ref_p).abs()
        check("out step JF=%d mode=%d halves=%d flags=%d inpaint=%d" % (JF, mode, halves, flags, inpaint),
              (pred.t.double() - ref_p).abs(), bound.view(B, T, JF).permute(0, 2, 1), mutants,
              where=~mask if inpaint else None)
        if inpaint:
            assert torch.equal(pred.t[mask], (motion.clamp(-1, 1) if flags & CLIP else motion)[mask])
        check_x_out(mode, pred.t, xt, noise, xout.t)


# ------------------------------------------------------------------------------------------------ DPM-Solver++
@pytest.mark.parametrize("JF", WIDTHS)
def test_out_dpm_width(JF):
    """EpiOut<OutDpm> at width JF, orders 1 and 2 at a second-order step: x_out bit for bit against the fp32 update from
    the engine's x0, the history slot k written with that x0 and nothing else of the history touched."""
    lib = _lib.load()
    diffusion = rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(1000, "20"), betas=gd.get_named_beta_schedule("cosine", 1000),
                                   model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_SMALL,
                                   loss_type=gd.LossType.MSE)
    table = diffusion.schedule_dpm_rows()
    i, k = 9, 10
    B, T, s_off, halves = 4, 40, 1, 2
    for order in (1, 2):
        g = torch.Generator(device="cuda").manual_seed(JF * 10 + order)
        _, _, hres, scale, w, b, xt = _inputs(g, B, JF, T, halves, s_off)
        n = B * JF * T
        hist = Guarded((2, B, JF, T), sample=JF * T)
        init = torch.randn(2, B, JF, T, device="cuda", generator=g)
        hist.t.copy_(init)
        before = hist.buf.clone()
        out = Guarded((B, JF, T), sample=JF * T)
        row = torch.from_numpy(table[i]).cuda()
        _lib.check(lib.b200mdm_test_out_dpm(_p(hres), _p(scale), _p(w), _p(b), _p(xt), _p(row), i, k, order, 0, None, None,
                                            _p(hist.t), _p(out.t), B, JF, T, D, s_off, halves, _stream()))
        torch.cuda.synchronize()
        out.check("x_out JF=%d order=%d" % (JF, order))
        x0 = _x0(lib, hres, scale, w, b, xt, 0, None, None, s_off, halves)
        assert torch.equal(hist.t[k % 2], x0)
        changed = hist.buf != before
        lo = hist.g + (k % 2) * n
        assert int(changed[:lo].sum() + changed[lo + n:].sum()) == 0, "history outside slot k written"
        second = order == 2
        want = do.update32(table[i], xt.cpu().numpy(), x0.cpu().numpy(), init[(k - 1) % 2].cpu().numpy() if second else None)
        got = out.t.cpu().numpy()
        assert np.array_equal(got, want), (order, np.abs(got - want).max())
        if second:
            assert not np.array_equal(got, do.update32(table[i][[0, 1, 3, 2]], xt.cpu().numpy(), x0.cpu().numpy(),
                                                       init[(k - 1) % 2].cpu().numpy()))
        print("  out dpm JF=%d order=%d: x_out bit-exact" % (JF, order))


# ------------------------------------------------------------------------------------------------ variational bound
@pytest.mark.parametrize("JF", WIDTHS)
def test_out_vb_width(JF):
    """EpiOut<OutVb> + vb_reduce_kernel at width JF, at i = 0 (the decoder term) and a middle index (FIXED_LARGE, so the
    KL term of a zero element is not zero): the per-element terms bit for bit against the fp32 restatement, the reduced
    means bit for bit against the engine-order restatement and within the fp32 summation bound of the fp64 mean over
    exactly JF * T elements; the mutants of the chunk geometry must miss that bound by MUTANT_MARGIN."""
    lib = _lib.load()
    diffusion = rs.SpacedDiffusion(use_timesteps=rs.space_timesteps(1000, "20"), betas=gd.get_named_beta_schedule("cosine", 1000),
                                   model_mean_type=gd.ModelMeanType.START_X, model_var_type=gd.ModelVarType.FIXED_LARGE,
                                   loss_type=gd.LossType.MSE)
    table = diffusion.schedule_vb_rows()
    n = diffusion.num_timesteps
    _, _, N, nc, _ = geometry(JF)
    B, T, s_off, halves = 3, 40, 1, 2
    for i in (0, 9):
        g = torch.Generator(device="cuda").manual_seed(JF * 10 + i)
        _, _, hres, scale, w, b, _ = _inputs(g, B, JF, T, halves, s_off)
        xs = nan_tail(torch.randn(B, JF, T, device="cuda", generator=g), JF * T)
        nz = nan_tail(torch.randn(B, JF, T, device="cuda", generator=g), JF * T)
        xt = nan_tail(torch.tensor(np.float32(table[i, 6]), device="cuda") * xs
                      + torch.tensor(np.float32(table[i, 7]), device="cuda") * nz, JF * T)
        row = torch.from_numpy(table[i]).cuda()
        elem = Guarded((3, B, JF, T), sample=JF * T)
        terms = Guarded((3, B, n))
        pred = Guarded((B, JF, T), sample=JF * T)
        _lib.check(lib.b200mdm_test_out_vb(_p(hres), _p(scale), _p(w), _p(b), _p(xt), _p(xs), _p(nz), _p(row), i, n, 0,
                                           None, None, _p(pred.t), _p(elem.t), _p(terms.t), B, JF, T, D, s_off, halves,
                                           _stream()))
        torch.cuda.synchronize()
        col = n - 1 - i
        live = torch.zeros(3, B, n, dtype=torch.bool, device="cuda")
        live[:, :, col] = True
        elem.check("vb elements JF=%d i=%d" % (JF, i))
        pred.check("vb pred_xstart JF=%d i=%d" % (JF, i))
        terms.check("vb terms JF=%d i=%d" % (JF, i), live)
        x0 = _x0(lib, hres, scale, w, b, xt, 0, None, None, s_off, halves)
        assert torch.equal(pred.t, x0)
        want = torch.stack(_restate(table[i], xs, xt, x0, nz, i == 0))
        assert torch.equal(elem.t, want), float((elem.t - want).abs().max())
        got = terms.t[:, :, col].double()
        engine_order = torch.stack([vo.engine_mean(want[0].cpu(), True), vo.engine_mean(want[1].cpu()),
                                    vo.engine_mean(want[2].cpu())])
        assert torch.equal(got.float().cpu(), engine_order)
        # fp64 mean over exactly JF * T elements; the kernel's fp32 sums: 32 columns of a chunk, ceil(T nc / 256) slots
        # of a lane, the 8-level tree, the division by the count and, for vb, by log 2
        e64 = elem.t.double().reshape(3, B, -1)
        scl = torch.tensor([1 / math.log(2), 1.0, 1.0], dtype=torch.float64, device="cuda")[:, None]
        ref = e64.mean(-1) * scl
        depth = 32 + -(-T * nc // 256) + 8
        bound = depth * U32 * e64.abs().mean(-1) * scl + 3 * U32 * ref.abs()
        mutants = {}
        if 32 * nc != JF:
            mutants["count 32 * vb_chunks * T"] = (ref * JF / (32 * nc) - ref).abs()
        if N != JF:
            mutants["count N_out * T"] = (ref * JF / N - ref).abs()
            z = torch.zeros(1, device="cuda")
            dead = _restate(table[i], z, z, z, z, i == 0)[0].double()      # the term of a zero-input dead column
            dv = torch.zeros_like(ref)
            dv[0] = (N - JF) / JF * dead / math.log(2)
            mutants["dead columns' terms in the sums"] = dv.abs()
        check("vb means JF=%d i=%d" % (JF, i), (got - ref).abs(), bound, mutants)


# ------------------------------------------------------------------------------------------------ soft inpainting
@pytest.mark.parametrize("JF", WIDTHS)
def test_out_weight_width(JF):
    """The weighted x0 of every update family's epilogue at width JF, with fractional, 0 and 1 weights: bit for bit
    against the fp32 restatement, written exactly."""
    lib = _lib.load()
    B, T, s_off, halves = 3, 40, 1, 2
    g = torch.Generator(device="cuda").manual_seed(JF)
    _, _, hres, scale, w_out, b_out, xt = _inputs(g, B, JF, T, halves, s_off)
    motion = nan_tail(torch.rand(B, JF, T, device="cuda", generator=g) * 2.4 - 1.2, JF * T)
    w = torch.rand(B, JF, T, device="cuda", generator=g)
    w[:, :, :6] = 0.0
    w[:, :, 6:12] = 1.0
    w[:, JF - 1, 12:18] = 0.0
    w[:, JF // 2, 18:24] = 1.0
    w = nan_tail(w, JF * T)
    for mode in FAMILIES:
        for clip in ((False, True) if mode == _lib.MODE_X0 else (False,)):
            def x0(weight, flags):
                out = Guarded((B, JF, T), sample=JF * T)
                _lib.check(lib.b200mdm_test_out_weight(_p(hres), _p(scale), _p(w_out), _p(b_out), _p(xt), mode, flags,
                                                       _p(weight), _p(motion if weight is not None else None), _p(out.t),
                                                       B, JF, T, D, s_off, halves, _stream()))
                torch.cuda.synchronize()
                out.check("weighted x0 JF=%d mode=%d" % (JF, mode))
                return out.t
            raw = x0(None, 0)
            got = x0(w, _lib.FLAG_CLIP_DENOISED if clip else 0)
            want = dt.soft_inpaint(raw, w, motion, clip=clip)
            assert torch.equal(got, want), (mode, clip, float((got - want).abs().max()))
            assert not torch.equal(got, dt.soft_inpaint(raw, w, motion, swap=True, clip=clip))
    print("  weighted x0 JF=%d: %d families bit-exact" % (JF, len(FAMILIES)))


# ------------------------------------------------------------------------------------------------ the engine at 251
def _kit_model(c, guided=True):
    args, sdkw = gk.kit_args(c)
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(**sdkw)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    assert model.engine().cfg.njoints * model.engine().cfg.nfeats == gk.KIT_JF
    return (b200mdm.ClassifierFreeSampleModel(model) if guided else model), model, diffusion, sd


def _y(inp, scale=True, **extra):
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), text_embed=inp["text_embed"].cuda(), **extra)
    if scale:
        y["scale"] = inp["scale"].cuda()
    return y


def _report(name, e):
    print("  %s: relative error vs the reference %.2e" % (name, e))
    assert e < RTOL, (name, e)


def test_kit_fixture_parity(golden):
    """Every forward and loop of kit_small.npz (the unmodified reference at 251 features) within 1e-3; the t = 0 bound
    column and the prior as test_vb_gpu.py checks them; graph and eager loops bit-identical."""
    gf = golden("kit_small.npz")
    c = gk.KIT
    cfg, model, diffusion, _ = _kit_model(c)
    inp = gk.kit_inputs(c)
    B, T = c["B"], c["T"]
    shape = (B, gk.KIT_JF, 1, T)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    t = torch.full((B,), c["t_fwd"], dtype=torch.long, device="cuda")
    with torch.no_grad():
        _report("fwd_cond", rel_err(model(xT, t, y=_y(inp, False)).cpu(), gf["kit_fwd_cond"]))
        _report("fwd_uncond", rel_err(model(xT, t, y=_y(inp, False, uncond=True)).cpu(), gf["kit_fwd_uncond"]))
        _report("fwd_cfg", rel_err(cfg(xT, t, y=_y(inp)).cpu(), gf["kit_fwd_cfg"]))
    y = _y(inp)
    prog = [o["sample"].clone() for o in diffusion.p_sample_loop_progressive(cfg, shape, noise=xT, clip_denoised=False,
                                                                             model_kwargs={"y": y}, noise_tape=tape)]
    for k, want in enumerate(gf["kit_ddpm_steps"]):
        _report("ddpm step %d" % k, rel_err(prog[k].cpu(), want))
    loops = {}
    for use_graph in (True, False):
        loops[use_graph] = diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y},
                                                   noise_tape=tape, use_graph=use_graph)
    assert torch.equal(loops[True], loops[False]) and torch.equal(loops[True], prog[-1])
    for eta in (0.0, 0.5):
        runs = [diffusion.ddim_sample_loop(cfg, shape, noise=xT, clip_denoised=False, eta=eta, model_kwargs={"y": y},
                                           noise_tape=tape, use_graph=ug) for ug in (True, False)]
        assert torch.equal(runs[0], runs[1])
        _report("ddim eta %g" % eta, rel_err(runs[0].cpu(), gf["kit_ddim_eta%g" % eta]))
    pcfg, _, pdiff, _ = _kit_model(dict(c, steps=gk.PLMS_STEPS))
    runs = [pdiff.plms_sample_loop(pcfg, shape, noise=xT, clip_denoised=False, model_kwargs={"y": y}, order=2,
                                   use_graph=ug) for ug in (True, False)]
    assert torch.equal(runs[0], runs[1])
    _report("plms (%d steps)" % gk.PLMS_STEPS, rel_err(runs[0].cpu(), gf["kit_plms"]))
    mask, motion = gk.kit_inpaint(c)
    yi = _y(inp, inpainting_mask=mask.cuda(), inpainted_motion=motion.cuda())
    o = diffusion.p_sample_loop(cfg, shape, noise=xT, clip_denoised=True, model_kwargs={"y": yi}, noise_tape=tape)
    _report("ddpm clip + inpaint", rel_err(o.cpu(), gf["kit_ddpm_clip_inpaint"]))
    runs = [diffusion.calc_bpd_loop(cfg, xT, clip_denoised=False, model_kwargs={"y": y}, noise_tape=tape, use_graph=ug)
            for ug in (True, False)]
    for k in gk.BPD_KEYS:
        assert torch.equal(runs[0][k], runs[1][k]), k
    r = runs[0]
    want = {k: torch.from_numpy(gf["kit_bpd_" + k]) for k in gk.BPD_KEYS}
    for k in ("xstart_mse", "mse"):
        _report("bpd " + k, rel_err(r[k].cpu(), want[k]))
    _report("bpd vb t>0", rel_err(r["vb"][:, :-1].cpu(), want["vb"][:, :-1]))
    perr = (r["prior_bpd"].cpu().double() - want["prior_bpd"].double()).abs()
    assert torch.all(perr <= RTOL * want["prior_bpd"].double().abs() + 2.0 ** -23 / math.log(2.0)), perr
    xt0 = (torch.tensor(np.float32(diffusion.sqrt_alphas_cumprod[0]), device="cuda") * xT
           + torch.tensor(np.float32(diffusion.sqrt_one_minus_alphas_cumprod[0]), device="cuda") * tape[-1])
    x0 = diffusion.p_mean_variance(cfg, xt0, torch.zeros(B, dtype=torch.long, device="cuda"), clip_denoised=False,
                                   model_kwargs={"y": y})["pred_xstart"]
    f64, bound = _t0_bound(diffusion, xT, xt0, x0)
    err = (r["vb"][:, -1].cpu().double() - f64).abs()
    print("  bpd t=0: |engine - fp64| %s, bound %s" % (err.numpy(), bound.numpy()))
    assert torch.all(err <= bound), (err, bound)
    assert torch.all((want["vb"][:, -1].double() - r["vb"][:, -1].cpu().double()).abs() <= T0_ABS_BITS)
    _report("total_bpd", rel_err(r["total_bpd"].cpu(), want["total_bpd"]))


def test_kit196_and_uestc_parity(golden):
    gf = golden("kit_small.npz")
    c = gk.KIT196
    cfg, _, diffusion, _ = _kit_model(c)
    inp = gk.kit_inputs(c)
    xT, tape = inp["tape"][0].cuda(), torch.stack(inp["tape"][1:]).cuda()
    with torch.no_grad():
        t = torch.full((c["B"],), c["t_fwd"], dtype=torch.long, device="cuda")
        _report("T=196 fwd_cfg", rel_err(cfg(xT, t, y=_y(inp)).cpu(), gf["kit196_fwd_cfg"]))
    o = diffusion.p_sample_loop(cfg, (c["B"], gk.KIT_JF, 1, c["T"]), noise=xT, clip_denoised=False,
                                model_kwargs={"y": _y(inp)}, noise_tape=tape)
    _report("T=196 ddpm", rel_err(o.cpu(), gf["kit196_ddpm"]))
    u = gk.UESTC
    args, sdkw = gk.uestc_args()
    model, diffusion = b200mdm.create_model_and_diffusion(args, SimpleNamespace(dataset=SimpleNamespace(num_actions=40)))
    b200mdm.load_model_wo_clip(model, b200mdm.synthetic_state_dict(**sdkw))
    model.to("cuda").eval()
    inp, action = gk.uestc_inputs()
    y = dict(mask=inp["mask"].cuda(), lengths=inp["lengths"].cuda(), action=action.cuda())
    o = diffusion.p_sample_loop(model, (u["B"], 25, 6, u["T"]), noise=inp["tape"][0].cuda(), clip_denoised=False,
                                model_kwargs={"y": y}, noise_tape=torch.stack(inp["tape"][1:]).cuda())
    _report("uestc 40 actions", rel_err(o.cpu(), gf["uestc_sample"]))


def _small():
    c = dict(gk.KIT, steps=6, B=3, T=24, lengths=[24, 17, 1], scales=[2.5, 1.0, 0.0], weights_seed=87, inputs_seed=88)
    cfg, _, diffusion, sd = _kit_model(c)
    inp = gk.kit_inputs(c)
    W = mo.OracleWeights(sd, c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    f = po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], inp["lengths"])
    return c, cfg, diffusion, inp, tabs, f


def test_kit_dpm_solver_vs_oracle():
    c, cfg, diffusion, inp, tabs, f = _small()
    shape = (c["B"], gk.KIT_JF, 1, c["T"])
    steps = [o["sample"].clone() for o in diffusion.dpm_solver_sample_loop_progressive(
        cfg, shape, noise=inp["tape"][0].cuda(), clip_denoised=False, model_kwargs={"y": _y(inp)}, order=2)]
    ref = []
    do.dpm_loop(f, tabs, inp["tape"][0], order=2, collect=ref)
    errs = [rel_err(s.cpu(), r) for s, (r, _) in zip(steps, ref)]
    print("  KIT DPM-Solver++(2M) per step: %s" % " ".join("%.2e" % e for e in errs))
    assert len(steps) == len(ref) and max(errs) < RTOL


def test_kit_ddim_inversion_vs_oracle():
    c, cfg, diffusion, inp, tabs, f = _small()
    x = inp["tape"][1].cuda()
    steps = [o["sample"].clone() for o in diffusion.ddim_reverse_sample_loop_progressive(
        cfg, x, clip_denoised=False, model_kwargs={"y": _y(inp)})]
    ref = []
    ro.reverse_loop(f, tabs, inp["tape"][1], collect=ref)
    errs = [rel_err(s.cpu(), r) for s, (r, _) in zip(steps, ref)]
    print("  KIT DDIM inversion per step: %s" % " ".join("%.2e" % e for e in errs))
    assert len(steps) == len(ref) and max(errs) < RTOL


def test_kit_headline_shape():
    """B = 64, T = 196, L = 8, guidance 2.5, 50 DDIM steps at 251 features: 3 samples against the fp32 oracle."""
    L, steps, B, T = 8, 50, 64, 196
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(dataset="kit", layers=L, diffusion_steps=steps),
                                                          SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(num_layers=L, input_feats=gk.KIT_JF, seed=89)
    b200mdm.load_model_wo_clip(model, sd)
    cfg = b200mdm.ClassifierFreeSampleModel(model.to("cuda").eval())
    inp = b200mdm.synthetic_inputs(B, njoints=gk.KIT_JF, nframes=T, steps=steps, seed=90, scale=torch.full((B,), 2.5),
                                   lengths=[T - 3 * (b % 40) for b in range(B)])
    tape = torch.stack(inp["tape"][1:]).cuda()
    out = diffusion.ddim_sample_loop(cfg, (B, gk.KIT_JF, 1, T), noise=inp["tape"][0].cuda(), clip_denoised=False, eta=0.0,
                                     model_kwargs={"y": _y(inp)}, noise_tape=tape).cpu()
    S = 3
    W = mo.OracleWeights(sd, L)
    tabs = so.diffusion_tables(so.named_betas("cosine", steps))
    with torch.no_grad():
        want = mo.sample_loop(W, tabs, list(range(steps)), [e[:S] for e in inp["tape"]], inp["text_embed"][:, :S],
                              inp["scale"][:S], inp["lengths"][:S], sampler="ddim")
    e = rel_err_per_sample(out[:S], want)
    print("  KIT headline, per sample vs the fp32 oracle: %s" % " ".join("%.2e" % v for v in e.tolist()))
    assert (e < RTOL).all()


def test_kit_handshake_ddim_vs_oracle():
    """HandshakeSampleModel (h = 4) over 2 motions of 2 windows at 251 features, DDIM against handshake_oracle."""
    c = dict(gk.KIT, steps=6, B=4, T=24, lengths=[24, 20, 24, 22], scales=[2.5, 1.0, 2.5, 0.0], weights_seed=91,
             inputs_seed=92)
    h, starts = 4, torch.tensor([True, False, True, False])
    cfg, _, diffusion, sd = _kit_model(c)
    inp = gk.kit_inputs(c)
    y = _y(inp, motion_start=starts.cuda())
    out = diffusion.ddim_sample_loop(b200mdm.HandshakeSampleModel(cfg, h), (c["B"], gk.KIT_JF, 1, c["T"]),
                                     noise=inp["tape"][0].cuda(), clip_denoised=False, eta=0.0, model_kwargs={"y": y},
                                     noise_tape=torch.stack(inp["tape"][1:]).cuda())
    W = mo.OracleWeights(sd, c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    den = ho.denoiser(po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], inp["lengths"]), h,
                      inp["lengths"], starts)
    with torch.no_grad():
        ref = deo.sample_loop(den, tabs, inp["tape"], sampler="ddim")
    _report("handshake DDIM vs the fp32 oracle", rel_err(out.cpu(), ref))


def test_kit_soft_weighted_ddim_vs_oracle():
    """Soft inpainting weights (fractional, 0 and 1) in a DDIM loop at 251 features against double_take_oracle."""
    c = dict(gk.KIT, steps=6, B=3, T=24, lengths=[24, 17, 24], scales=[2.5, 1.0, 0.0], weights_seed=93, inputs_seed=94)
    cfg, _, diffusion, sd = _kit_model(c)
    inp = gk.kit_inputs(c)
    shape = (c["B"], gk.KIT_JF, 1, c["T"])
    g = torch.Generator().manual_seed(95)
    weight = torch.rand(shape, generator=g)
    weight[..., :4] = 1.0
    weight[..., 4:8] = 0.0
    weight[:, -1] = 1.0                                        # the last live column of the last live chunk
    motion = torch.rand(shape, generator=g) * 2 - 1
    y = _y(inp, inpainting_weight=weight.cuda(), inpainted_motion=motion.cuda())
    out = diffusion.ddim_sample_loop(cfg, shape, noise=inp["tape"][0].cuda(), clip_denoised=False, eta=0.0,
                                     model_kwargs={"y": y}, noise_tape=torch.stack(inp["tape"][1:]).cuda())
    W = mo.OracleWeights(sd, c["L"])
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    den = dt.denoiser(po.enc_denoiser(W, list(range(c["steps"])), inp["text_embed"], inp["scale"], inp["lengths"]),
                      weight, motion)
    with torch.no_grad():
        ref = deo.sample_loop(den, tabs, inp["tape"], sampler="ddim")
    _report("soft-weighted DDIM vs the fp32 oracle", rel_err(out.cpu(), ref))


def test_kit_dip_chain_vs_oracle():
    """DiP's autoregressive chain at 251 features: each chunk's prefix handed over on the device (chain_handoff_kernel,
    then pack_input at row 0), 3 chunks against the fp32 oracle."""
    chain_against_fp32_oracle(*build_chain(dataset="kit"), gk.KIT_JF)
