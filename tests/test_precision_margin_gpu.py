"""GPU: full-depth (L = 8) guided forwards and 10-step DDIM loops of the four model kinds of tests/precision_cases.py
(trans_enc text with CFG, a2m without it, DiP, the CLIP decoder), per sample, under the weight families of
oracle/weight_families.py (init scale, sharper attention, larger FFN activations, LayerNorm bias outliers).

  (a) Engine vs the site-exact fp16 emulation (mdm_oracle.Sites: fp16 exactly where the engine keeps fp16): a coarse
      sanity check only.  Two fp16 pipelines that differ only in fp32 accumulation order do not track each other over
      8 layers: where an fp32 value lies near an fp16 rounding boundary, one fp32 ulp flips the rounding, and the flips
      compound at every rounding site downstream.  The emulation run on an input with one fp32 ulp of random relative
      noise moves from itself as far as the engine is from it, and so does an emulation with one site wrong (q / k or P
      left in fp32), so this cannot tell such a fault apart; the kernel tests against fp64 do.  The engine must stay
      within EMU_SLACK of that spread.
  (b) Engine vs the fp32 oracle, 1e-3 per sample on every loop sample of the init-scale weights (the documented
      contract, test_init_loop_per_sample).
  (c) Engine vs the fp32 oracle on every output and family: no worse than 1.25 x the emulation + 1e-5.
(a) and (c) are skipped for an output whose emulation is more than CHAOTIC from fp32 (the 10-step loops of the
sharpest family drift to O(1) differences, where two results are effectively independent).  Every error is a
per-sample Frobenius ratio (rel_err_per_sample): one bad sample is not diluted by the batch.  Each case prints its
layer-0 statistics and, per output, the errors of each sample (DESIGN.md section 2 records them)."""
import pytest
import torch

from oracle import mdm_oracle as mo, weight_families as wf
from precision_cases import KINDS, L, T_HI, T_LO, fmt, rel_err_per_sample, ulp_noise

pytestmark = pytest.mark.gpu
RTOL = 1e-3
EMU_SLACK = 3.0
CHAOTIC = 0.1


@pytest.mark.parametrize("family", wf.FAMILIES)
@pytest.mark.parametrize("kind", list(KINDS))
def test_precision_margin(kind, family):
    k = KINDS[kind]()
    sd, st = wf.family_state_dict(family, k.make_sd, k.probe)
    forward, loop = k.engine(sd)
    W = mo.OracleWeights(sd, L)
    x, tape = k.inp["tape"][0], k.inp["tape"]
    got = {T_HI: forward(x, T_HI), T_LO: forward(x, T_LO), "loop": loop()}
    print("\n%s / %s: layer 0 %s" % (kind, family, ", ".join("%s %.4g" % kv for kv in st.items())))
    bad = []
    with torch.no_grad():
        for key, out in got.items():
            def ref(cast, noisy=False, key=key):
                if key == "loop":
                    return k.loop(W, cast, [ulp_noise(tape[0])] + tape[1:] if noisy else tape)
                return k.forward(W, ulp_noise(x) if noisy else x, key, cast)
            name = "ddim loop" if key == "loop" else "forward t=%d" % key
            f32, emu = ref(None), ref(k.sites)
            e_emu, e_f32, emu_f32 = rel_err_per_sample(out, emu), rel_err_per_sample(out, f32), rel_err_per_sample(emu, f32)
            spread = rel_err_per_sample(ref(k.sites, noisy=True), emu)
            chaotic = emu_f32.max() > CHAOTIC
            print("  %-12s engine-fp32 %s  emulation-fp32 %s  engine-emulation %s  emulation spread %s%s" % (
                name, fmt(e_f32), fmt(emu_f32), fmt(e_emu), fmt(spread), "  (chaotic: not checked)" if chaotic else ""))
            if chaotic:
                continue
            if not e_emu.max() <= EMU_SLACK * spread.max() + 1e-5:
                bad.append("(a) %s: engine vs emulation %s, emulation spread %s" % (name, fmt(e_emu), fmt(spread)))
            if not (e_f32 <= 1.25 * emu_f32 + 1e-5).all():
                bad.append("(c) %s: engine vs fp32 %s, emulation vs fp32 %s" % (name, fmt(e_f32), fmt(emu_f32)))
    assert not bad, "\n".join(bad)


ENC_GUIDANCE_7_5 = pytest.mark.xfail(strict=True, reason=(
    "open contract violation: the guidance-7.5 sample measures 2.07e-3 against fp32 on an H100 (the site-exact fp16 "
    "emulation 2.09e-3), from the encoder's fp16 attention output, FFN-up input and GELU output; keeping all three in "
    "[hi | lo], as DiP does, gives 5.0e-4 in the emulation (DESIGN.md section 2)"))


@pytest.mark.parametrize("kind", [pytest.param(k, marks=ENC_GUIDANCE_7_5) if k == "trans_enc_text" else k for k in KINDS])
def test_init_loop_per_sample(kind):
    """(b): a 10-step DDIM loop on the init-scale weights holds 1e-3 against the fp32 oracle on every sample."""
    k = KINDS[kind]()
    sd = k.make_sd()
    _, loop = k.engine(sd)
    with torch.no_grad():
        want = k.loop(mo.OracleWeights(sd, L), None, k.inp["tape"])
    e = rel_err_per_sample(loop(), want)
    print("%s init, 10-step DDIM loop: engine vs fp32 per sample %s" % (kind, fmt(e)))
    assert (e <= RTOL).all(), fmt(e)
