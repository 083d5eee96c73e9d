"""CPU: the long-text-memory fixture (tests/golden/dip_longmem_small.npz, made by oracle/gen_golden_longmem.py from the
unmodified reference): the fp32 oracle reproduces it, and so does the generator."""
import numpy as np
import pytest
import torch

import b200mdm
from conftest import rel_err
from oracle import gen_golden_longmem as gl
from oracle import mdm_oracle as mo
from oracle import ref_harness as rh
from oracle import schedule_oracle as so

TOL = 2e-5


def test_oracle_reproduces_dip_longmem(golden):
    g = golden("dip_longmem_small.npz")
    c = gl.DIP
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                      seed=c["weights_seed"]), c["L"])
    inp, enc, tmask, prefix = gl.dip_inputs()
    assert enc.shape[0] == 150 and tmask.any(1).tolist() == [False, True, True]
    out = mo.cfg_denoise_dec(W, inp["tape"][0], 1, enc, tmask, prefix, inp["scale"], inp["lengths"])
    assert rel_err(out, g["dip_fwd_cfg"]) < TOL
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    o = mo.sample_loop_dec(W, tabs, list(range(c["steps"])), inp["tape"], enc, tmask, prefix, inp["scale"], inp["lengths"])
    assert rel_err(o, g["dip_ddpm"]) < TOL


def test_oracle_reproduces_bert_decoder_longmem(golden):
    g = golden("dip_longmem_small.npz")
    c = gl.BERT
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=c["L"], cond_dim=768,
                                                      seed=c["weights_seed"]), c["L"])
    inp, enc, tmask = gl.bert_inputs()
    tabs = so.diffusion_tables(so.named_betas("cosine", c["steps"]))
    o = mo.sample_loop_dec(W, tabs, list(range(c["steps"])), inp["tape"], enc, tmask, torch.zeros(c["B"], 263, 1, 0),
                           inp["scale"], inp["lengths"])
    assert rel_err(o, g["bert_ddpm"]) < TOL


@pytest.mark.skipif(not rh.available(), reason="reference tree not present")
def test_golden_reproduces_from_generator(golden, tmp_path, monkeypatch):
    """The generator pins the reference to gl.THREADS intra-op threads, so this holds on any core count."""
    g = golden("dip_longmem_small.npz")
    monkeypatch.setattr(gl, "OUT", str(tmp_path))
    threads = torch.get_num_threads()
    new = gl.gen_longmem_small()
    assert torch.get_num_threads() == threads
    assert set(new) == set(g.files)
    for k in g.files:
        if k != "meta":
            np.testing.assert_allclose(new[k], g[k], rtol=1e-6, atol=1e-6, err_msg=k)
