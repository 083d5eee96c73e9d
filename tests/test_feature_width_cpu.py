"""CPU: the fp32 oracles (oracle/mdm_oracle.py, plms_oracle.py, vb_oracle.py) at the feature widths of KIT (251) and
UESTC (25 x 6 = 150 with 40 action classes), against tests/golden/kit_small.npz, which the unmodified reference produced
(oracle/gen_golden_kit.py).  Tolerances as in tests/test_oracle_cpu.py and tests/test_vb_cpu.py."""
import numpy as np
import torch

import b200mdm
from conftest import rel_err
from oracle import gen_golden_kit as gk
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import schedule_oracle as so
from oracle import vb_oracle as vo

TOL = 2e-5
RTOL_BPD = 1e-3


def kit_setup(c):
    """(oracle weights, inputs, fp64 tables, timestep map) of a KIT case of the fixture."""
    _, sdkw = gk.kit_args(c)
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(**sdkw), c["L"])
    return W, gk.kit_inputs(c), so.diffusion_tables(so.named_betas("cosine", c["steps"])), list(range(c["steps"]))


def clip_inpaint_loop(denoise, tabs, tape, inpaint):
    """p_sample_loop with clip_denoised=True: inpainting blend, then clamp, then the DDPM step (the reference's order)."""
    x = tape[0].clone()
    n = len(tabs["betas"])
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = po.p_mean_x0(denoise(x, i), True, inpaint)
        x, _ = mo.p_sample_step(tabs, x0, x, i, tape[1 + k])
    return x


def test_kit_widths(golden):
    g = golden("kit_small.npz")
    for key in ("kit_fwd_cfg", "kit_ddpm_steps", "kit196_ddpm"):
        assert g[key].shape[-3:-1] == (gk.KIT_JF, 1), key
    assert g["uestc_sample"].shape[1:3] == (25, 6)


def test_kit_forwards(golden):
    g = golden("kit_small.npz")
    c = gk.KIT
    W, inp, _, _ = kit_setup(c)
    x, te, ln = inp["tape"][0], inp["text_embed"], inp["lengths"]
    assert rel_err(mo.denoise_enc(W, x, c["t_fwd"], te, ln), g["kit_fwd_cond"]) < TOL
    assert rel_err(mo.denoise_enc(W, x, c["t_fwd"], te, ln, uncond=True), g["kit_fwd_uncond"]) < TOL
    assert rel_err(mo.cfg_denoise_enc(W, x, c["t_fwd"], te, inp["scale"], ln), g["kit_fwd_cfg"]) < TOL


def test_kit_loops(golden):
    g = golden("kit_small.npz")
    c = gk.KIT
    W, inp, tabs, tmap = kit_setup(c)
    te, sc, ln = inp["text_embed"], inp["scale"], inp["lengths"]
    col = []
    mo.sample_loop(W, tabs, tmap, inp["tape"], te, sc, ln, collect=col)
    assert len(col) == len(g["kit_ddpm_steps"])
    for k, want in enumerate(g["kit_ddpm_steps"]):
        assert rel_err(col[k], want) < TOL, k
    for eta in (0.0, 0.5):
        o = mo.sample_loop(W, tabs, tmap, inp["tape"], te, sc, ln, sampler="ddim", eta=eta)
        assert rel_err(o, g["kit_ddim_eta%g" % eta]) < TOL, eta
    f = po.enc_denoiser(W, tmap, te, sc, ln)
    ptabs = so.diffusion_tables(so.named_betas("cosine", gk.PLMS_STEPS))
    fp = po.enc_denoiser(W, list(range(gk.PLMS_STEPS)), te, sc, ln)
    assert rel_err(po.plms_loop(fp, ptabs, inp["tape"][0], order=2), g["kit_plms"]) < TOL
    o = clip_inpaint_loop(f, tabs, inp["tape"], gk.kit_inpaint(c))
    assert rel_err(o, g["kit_ddpm_clip_inpaint"]) < TOL


def test_kit_bpd(golden):
    g = golden("kit_small.npz")
    W, inp, tabs, tmap = kit_setup(gk.KIT)
    f = po.enc_denoiser(W, tmap, inp["text_embed"], inp["scale"], inp["lengths"])
    with torch.no_grad():
        got = vo.vb_loop(f, tabs, inp["tape"][0], inp["tape"][1:], False)
    for k in gk.BPD_KEYS:
        want = torch.from_numpy(g["kit_bpd_" + k])
        e = rel_err(got[k], want)
        print("kit bpd %s: relative error vs the reference %.2e" % (k, e))
        assert got[k].shape == want.shape and e < RTOL_BPD, (k, e)


def test_kit196(golden):
    g = golden("kit_small.npz")
    c = gk.KIT196
    W, inp, tabs, tmap = kit_setup(c)
    te, sc, ln = inp["text_embed"], inp["scale"], inp["lengths"]
    assert rel_err(mo.cfg_denoise_enc(W, inp["tape"][0], c["t_fwd"], te, sc, ln), g["kit196_fwd_cfg"]) < TOL
    assert rel_err(mo.sample_loop(W, tabs, tmap, inp["tape"], te, sc, ln), g["kit196_ddpm"]) < TOL


def test_uestc_40_actions(golden):
    g = golden("kit_small.npz")
    c = gk.UESTC
    _, sdkw = gk.uestc_args()
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(**sdkw), c["L"])
    assert W["embed_action.action_embedding"].shape[0] == 40
    inp, action = gk.uestc_inputs()
    assert int(action.max()) == 39
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    o = mo.sample_loop(W, tabs, list(range(c["steps"])), inp["tape"], None, None, inp["lengths"], action=action)
    assert rel_err(o, g["uestc_sample"]) < TOL
    # the last class is a row of its own: the same run with action 38 for sample 0 moves that sample only
    o2 = mo.sample_loop(W, tabs, list(range(c["steps"])), inp["tape"], None, None, inp["lengths"],
                        action=torch.where(action == 39, 38, action))
    assert not torch.equal(o2[0], o[0]) and torch.equal(o2[1:], o[1:])
    assert np.isfinite(g["uestc_sample"]).all()
