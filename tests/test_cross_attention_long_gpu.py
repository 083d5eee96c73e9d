"""GPU: the long-memory cross-attention core (cross_attention_long_kernel: 64 < Mt <= 512, keys in blocks of 64 with an
online softmax) against an fp64 restatement of its blocked arithmetic, with a bound derived from that arithmetic and
host-side mutants that must miss it (check)."""
import pytest
import torch
import torch.nn.functional as F

from test_epilogues_gpu import U32, acc_bound, check, half_ulp16, split16
from test_kernels_gpu import CROSS_C, run_cross_attention

pytestmark = pytest.mark.gpu

KB = 64                        # keys per block
D, H, DH = 512, 4, 128
E2 = 2.0 ** -22                # exp2f: 2 ulp


def blocked(s, v, valid, rescale_o=True):
    """fp64 restatement of cross_attention_long_kernel for exact fp32 logits s [n, H, S, Mt] (raw q.k), v [n, H, Mt, dh]
    and the admitted keys valid [n, 1, 1, Mt].  Per block b of 64 keys: sc = fp32(s c) (-inf where not admitted),
    m_b = max(m_{b-1}, max of the block) in fp32, alpha_b = 2^fp32(m_{b-1} - m_b) (1 when m does not move),
    p = 2^fp32(sc - m_b) (offset 0 while m_b = -inf).  The kernel scales O and l by alpha_b before it adds block b, so
    in the final frame block b's p carries scale_b = prod_{b' > b} alpha_b'.
    Returns O (sum p v / l, fp64), A (sum p |v| / l), l and the per-block (p, scale) with v padded to whole blocks.
    rescale_o=False: the mutant that scales l but not O."""
    n, h, S, Mt = s.shape
    nb = (Mt + KB - 1) // KB
    pad = nb * KB - Mt
    sc = F.pad((s * CROSS_C).float().masked_fill(~valid, float("-inf")), (0, pad), value=float("-inf"))
    vp = F.pad(v, (0, 0, 0, pad))
    m = torch.full(sc.shape[:-1] + (1,), float("-inf"), device=s.device)
    ps, alphas = [], []
    for b in range(nb):
        blk = sc[..., b * KB:(b + 1) * KB]
        mn = torch.maximum(m, blk.amax(-1, keepdim=True))
        alphas.append(torch.where(mn == m, torch.ones_like(m, dtype=torch.float64), torch.exp2((m - mn).double())))
        off = torch.where(mn == float("-inf"), torch.zeros_like(mn), mn)
        ps.append(torch.exp2((blk - off).double()))
        m = mn
    scales, acc = [None] * nb, torch.ones_like(alphas[0])
    for b in reversed(range(nb)):
        scales[b] = acc
        acc = acc * alphas[b]
    pe = torch.cat([p * c for p, c in zip(ps, scales)], -1)
    l = pe.sum(-1, keepdim=True)
    num = pe @ vp if rescale_o else torch.cat(ps, -1) @ vp
    return num / l, (pe @ vp.abs()) / l, l, ps, scales, vp


def bound_of(s, v, valid):
    """O and the per-element bound on |kernel - O|.  Terms, first order (the factor 1 + 2^-16 covers the rest):
      * exp2f on every p and on each of up to nb - 1 alphas: 2^-22 relative apiece, in the numerator and in l;
      * O * alpha in fp32 before each later block: U32 of the partial sum (<= A l);
      * the fp16 split of P (lo rounded), p within 2^-22 of the emulated value, in the final frame;
      * the mma.sync accumulation in the kernel's order (per block, per 16 keys: hi products, then lo), in the
        final frame, where the rescaled partial sum is what each update rounds against;
      * l: per block 8 pair adds + 8 chain adds + scale and add per thread, then two quad shuffles, every partial
        <= l: U32 (18 nb + 2) l;
      * 1 / l and the product (IEEE), then half an fp16 ulp of O."""
    O, A, l, ps, scales, vp = blocked(s, v, valid)
    nb = len(ps)
    split, P2 = [], []
    for p, c in zip(ps, scales):
        pf = p.float()
        hi, lo = split16(pf)
        rem = (pf - hi.float()).double()
        split.append(torch.where(p > 0, half_ulp16(rem.abs() + E2 * p), torch.zeros_like(p)) * c)
        P2.append(torch.stack([(t.double() * c).view(*p.shape[:-1], KB // 16, 16) for t in (hi, lo)], -2)
                  .reshape(*p.shape[:-1], 2 * KB))
    P2 = torch.cat(P2, -1)
    vt = vp.transpose(-1, -2)
    V2 = torch.stack([vt.reshape(*vt.shape[:-1], nb * KB // 16, 16)] * 2, -2).reshape(*vt.shape[:-1], 2 * nb * KB)
    acc = acc_bound(P2, V2)
    e_split = torch.cat(split, -1) @ vp.abs()
    Oa = O.abs()
    rel_num = E2 * nb + U32 * (nb - 1)
    rel_l = E2 * nb + U32 * (18 * nb + 2)
    dO = (rel_num * A + (e_split + acc) / l + rel_l * Oa + 2 * U32 * Oa) * (1 + 2.0 ** -16)
    return O, dO + half_ulp16(Oa + dO), ps, scales, vp, l


def operands(n, S, Mt, ld, col0, seed):
    """q = integers in [-3, 3] (one sign per column of a sample and head), k = halves in [-2, 2]: every logit is exact
    in fp32 and the softmax keeps a handful of keys per row.  v = N(0, 1) in fp16."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sign = torch.randint(0, 2, (n, 1, H, DH), device="cuda", generator=g).float() * 2 - 1
    q = sign * torch.randint(0, 4, (n, S, H, DH), device="cuda", generator=g).float()
    k = torch.randint(-4, 5, (n, Mt, H, DH), device="cuda", generator=g).float() / 2
    kvw = torch.randn(n * Mt, ld, device="cuda", generator=g).half()
    return g, sign, q, k, kvw


def masks(n, Mt, g):
    """Per sample i mod 6: none; right padding (the BERT case); ragged; one whole 64-key block in the middle masked;
    only the last block valid; everything masked (must give exactly 0)."""
    nb = (Mt + KB - 1) // KB
    mask = torch.zeros(n, Mt, dtype=torch.bool, device="cuda")
    ragged = torch.rand(n, Mt, device="cuda", generator=g) < 0.3
    for i in range(n):
        kind = i % 6
        if kind == 1:
            mask[i, (3 * Mt) // 5:] = True
        elif kind == 2:
            mask[i, 1:] = ragged[i, 1:]
        elif kind == 3:
            b = nb // 2
            mask[i, b * KB:(b + 1) * KB] = True
        elif kind == 4:
            mask[i, :(nb - 1) * KB] = True
        elif kind == 5:
            mask[i] = True
    return mask


def heads(t, n, rows):                                                # [n * rows, d] -> [n, H, rows, dh]
    return t.double().view(n, rows, H, DH).permute(0, 2, 1, 3)


CASES = [(6, S, Mt, ld) for Mt in (65, 72, 127, 128, 129, 200, 256, 300, 511, 512)
         for S in (1, 17, 60, 61, 196, 197) for ld in (0, 7168)]
CASES += [(128, 60, 512, 7168), (128, 196, 130, 7168)]               # the engine's launch: 2 x 64 samples, layer 7


@pytest.mark.parametrize("n,S,Mt,ld_extra", CASES)
def test_cross_attention_long(n, S, Mt, ld_extra):
    """k | v sit at the end of a row of ld_extra more columns (the last layer's slice of the all-layer K/V projection).
    The last masked key of every partly masked sample carries the largest logit of each row (a wrong max would wipe
    out every admitted key), and the last admitted key of every sample is half aligned with the queries, so the
    running max usually grows in a late block (a missing rescale of O shows)."""
    ld, col0 = 2 * D + ld_extra, ld_extra
    g, sign, q, k, kvw = operands(n, S, Mt, ld, col0, 1000 * Mt + 10 * S + n + ld_extra)
    mask = masks(n, Mt, g)
    full = mask.all(1)
    padded = mask.any(1) & ~full
    key = torch.arange(Mt, device="cuda")
    last_pad = torch.where(mask, key, -1).amax(1)
    last_valid = torch.where(~mask, key, -1).amax(1)
    half = torch.rand(n, H, DH, device="cuda", generator=g) < 0.5
    for i in range(n):
        if padded[i]:
            k[i, last_pad[i]] = 2 * sign[i, 0]
        if not full[i]:
            k[i, last_valid[i]] = torch.where(half[i], sign[i, 0], k[i, last_valid[i]])
    kvw[:, col0:col0 + D] = k.reshape(n * Mt, D).half()
    q16 = q.reshape(n * S, D).half()
    out = run_cross_attention(q16, kvw, col0, mask, n, S, Mt)

    qq, kk, vv = heads(q16, n, S), heads(kvw[:, col0:col0 + D], n, Mt), heads(kvw[:, col0 + D:col0 + 2 * D], n, Mt)
    got = heads(out[:, :D], n, S)
    assert torch.equal(got[full], torch.zeros_like(got[full])), "a fully masked row must give 0"
    s = qq @ kk.transpose(-1, -2)                                     # exact: multiples of 1/2 below 2^11
    valid = (~mask)[:, None, None, :]
    O, bound, ps, scales, vp, l = bound_of(s, vv, valid)

    def rounded(o):
        return (torch.nan_to_num(o, nan=0.0).float().half().double() - O).abs()
    O_hi = torch.cat([split16(p.float())[0].double() * c for p, c in zip(ps, scales)], -1) @ vp / l
    admit = valid | ((key[None, :] == last_pad[:, None]) & padded[:, None])[:, None, None, :]
    drop = valid & (key[None, :] != last_valid[:, None])[:, None, None, :]
    mutants = {"last valid token dropped": rounded(blocked(s, vv, drop)[0]),
               "P hi only": rounded(O_hi),
               "padded token admitted": rounded(blocked(s, vv, admit)[0]),
               "rescale of O skipped when the max grows": rounded(blocked(s, vv, valid, rescale_o=False)[0])}
    where = ~full[:, None, None, None].expand_as(O)
    check("cross-attention long n=%d S=%d Mt=%d ld=%d" % (n, S, Mt, ld), (got - O).abs(), bound, mutants, where=where)


@pytest.mark.parametrize("S", [60, 196])
def test_padding_invariance(S):
    """40 admitted tokens right-padded to 300 through the long core against the same 40 unpadded through the short
    core (cross_attention_kernel<8>).  Both restate to the same fp64 O (the padded blocks leave the max and the scales
    alone), so the two outputs differ by at most the sum of their bounds."""
    n, Mv, Mt = 4, 40, 300
    g, sign, q, k, kvw = operands(n, S, Mt, 2 * D, 0, 7 * S)
    kvw[:, :D] = k.reshape(n * Mt, D).half()
    q16 = q.reshape(n * S, D).half()
    mask = torch.zeros(n, Mt, dtype=torch.bool, device="cuda")
    mask[:, Mv:] = True
    long = run_cross_attention(q16, kvw, 0, mask, n, S, Mt)
    kv_short = kvw.view(n, Mt, 2 * D)[:, :Mv].reshape(n * Mv, 2 * D).contiguous()
    short = run_cross_attention(q16, kv_short, 0, mask[:, :Mv], n, S, Mv)
    qq = heads(q16, n, S)
    kk, vv = heads(kvw[:, :D], n, Mt), heads(kvw[:, D:], n, Mt)
    s = qq @ kk.transpose(-1, -2)
    O_l, b_l = bound_of(s, vv, (~mask)[:, None, None, :])[:2]
    O_s, b_s = bound_of(s[..., :Mv], vv[:, :, :Mv], torch.ones(n, 1, 1, Mv, dtype=torch.bool, device="cuda"))[:2]
    err = (heads(long[:, :D], n, S) - heads(short[:, :D], n, S)).abs()
    r = (err / (b_l + b_s + (O_l - O_s).abs())).max().item()     # the last term: fp64 sums of different lengths
    print("padding invariance S=%d: |long - short| / (bound_long + bound_short) = %.3g" % (S, r))
    assert r <= 1.0
