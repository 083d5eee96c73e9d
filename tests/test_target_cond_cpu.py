"""CPU: target-location conditioning (multi_target_cond, model/mdm.py:64-73,197-199,399-480) -- parameter names and
shapes against the reference, the fp32 oracle against the reference's golden outputs, and the host-side handling of
the y keys (validation, sharding, the autoregressive sampler)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm.engine import canonical_target
from b200mdm.parallel import shard_model_kwargs
from conftest import default_args
from oracle import mdm_oracle as mo
from oracle import ref_harness as rh
from oracle import schedule_oracle as so
from oracle import target_oracle as to

JOINTS = b200mdm.synthetic.HML_TARGET_JOINTS
ENCODERS = [("single", 1), ("split", 2), ("multi", 1)]     # the layer counts target_keys.npz was made with


def _model(encoder, layers, arch="trans_enc"):
    over = dict(layers=1, multi_target_cond=True, multi_encoder_type=encoder, target_enc_layers=layers)
    if arch == "trans_dec":
        over.update(arch="trans_dec", text_encoder_type="bert", context_len=20, pred_len=40)
    model, _ = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    return model


def _target_items(sd):
    return {k: tuple(v.shape) for k, v in sd.items() if k.startswith("embed_target_cond.")}


@pytest.mark.parametrize("encoder,layers", ENCODERS)
@pytest.mark.parametrize("arch", ["trans_enc", "trans_dec"])
def test_keys_and_shapes_match_reference(golden, encoder, layers, arch):
    g = golden("target_keys.npz")
    ref = {k: tuple(int(s) for s in shp.split(",")) for k, shp in zip(g[encoder + "_names"], g[encoder + "_shapes"])}
    model = _model(encoder, layers, arch)
    assert _target_items(model.state_dict()) == ref
    assert model.extended_goal_joint_names == JOINTS
    sd = b200mdm.synthetic_state_dict(arch=arch, num_layers=1, cond_dim=768 if arch == "trans_dec" else 512,
                                      target_encoder=encoder, target_enc_layers=layers)
    assert _target_items(sd) == ref
    b200mdm.load_model_wo_clip(model, sd)


def test_target_params_leave_other_tensors_unchanged():
    plain = b200mdm.synthetic_state_dict(num_layers=2, seed=3)
    tgt = b200mdm.synthetic_state_dict(num_layers=2, seed=3, target_encoder="multi")
    assert set(tgt) - set(plain) == set(_target_items(tgt))
    assert all(torch.equal(plain[k], tgt[k]) for k in plain)


@pytest.mark.skipif(not rh.available(), reason="reference tree not present")
@pytest.mark.parametrize("encoder,layers", [("single", 2), ("split", 1), ("multi", 1)])
def test_reference_parameters_load(encoder, layers):
    over = dict(layers=1, multi_target_cond=True, multi_encoder_type=encoder, target_enc_layers=layers)
    ref_model, _ = rh.build(rh.default_args(**over))
    model = _model(encoder, layers)
    b200mdm.load_model_wo_clip(model, ref_model.state_dict())
    for k, v in _target_items(model.state_dict()).items():
        assert torch.equal(model.state_dict()[k], ref_model.state_dict()[k]), k


def test_still_unsupported_configs_raise():
    with pytest.raises(NotImplementedError):
        b200mdm.MDM(**b200mdm.get_model_args(default_args(layers=1, multi_target_cond=True, emb_policy="cat"),
                                             SimpleNamespace(dataset=SimpleNamespace())))
    with pytest.raises(ValueError):
        _model("bogus", 1)


def test_lambda_target_loc_implies_target_encoder():
    args = b200mdm.get_model_args(default_args(lambda_target_loc=1.0), SimpleNamespace(dataset=SimpleNamespace()))
    assert args["multi_target_cond"] is True
    args = b200mdm.get_model_args(default_args(), SimpleNamespace(dataset=SimpleNamespace()))
    assert args["multi_target_cond"] is False


def test_oracle_vs_golden(golden):
    tabs = so.diffusion_tables(so.named_betas("cosine", 3))
    tmap = np.arange(3)
    # DiP, single encoder
    g = golden("dip_target_small.npz")
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=2, cond_dim=768, seed=4,
                                                      target_encoder="single"), 2)
    enc, tmask, prefix = b200mdm.synthetic_dip_inputs(3, 7, 20)
    inp = b200mdm.synthetic_inputs(3, nframes=40, steps=3, seed=13, lengths=[40, 33, 12], scale=torch.tensor([7.5, 2.0, 1.0]))
    tg = b200mdm.synthetic_target_inputs(3, seed=5)
    valid = to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"])
    gt = to.target_embedding(W, "single", tg["target_cond"], valid)
    np.testing.assert_allclose(gt.numpy(), g["g"], rtol=1e-5, atol=1e-6)
    x = inp["tape"][0]
    args = (W, x, 1, enc, tmask, prefix)
    np.testing.assert_allclose(to.cfg(to.denoise_dec, inp["scale"], *args, gt, inp["lengths"]).numpy(), g["fwd_cfg"],
                               rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(to.cfg(to.denoise_dec, inp["scale"], *args, None, inp["lengths"]).numpy(),
                               g["fwd_cfg_target_uncond"], rtol=1e-4, atol=1e-4)
    out = to.sample_loop_dec(W, tabs, tmap, inp["tape"], enc, tmask, prefix, gt, inp["scale"], inp["lengths"])
    np.testing.assert_allclose(out.numpy(), g["ddpm"], rtol=1e-4, atol=1e-4)
    # trans_enc, multi encoder
    g = golden("enc_target_small.npz")
    W = mo.OracleWeights(b200mdm.synthetic_state_dict(num_layers=2, seed=6, target_encoder="multi"), 2)
    inp = b200mdm.synthetic_inputs(4, nframes=24, steps=3, seed=14, lengths=[24, 20, 11, 6],
                                   scale=torch.tensor([2.5, 1.0, 5.0, 2.5]))
    tg = b200mdm.synthetic_target_inputs(4, seed=8)
    valid = to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"])
    gt = to.target_embedding(W, "multi", tg["target_cond"], valid, joint_names=JOINTS)
    np.testing.assert_allclose(gt.numpy(), g["g"], rtol=1e-5, atol=1e-6)
    assert not gt[3].any()                                  # the empty joint set
    x = inp["tape"][0]
    np.testing.assert_allclose(to.denoise_enc(W, x, 2, inp["text_embed"], gt, inp["lengths"]).numpy(), g["fwd_cond"],
                               rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(to.cfg(to.denoise_enc, inp["scale"], W, x, 2, inp["text_embed"], gt, inp["lengths"]).numpy(),
                               g["fwd_cfg"], rtol=1e-4, atol=1e-4)
    out = to.sample_loop_enc(W, tabs, tmap, inp["tape"], inp["text_embed"], gt, inp["scale"], inp["lengths"])
    np.testing.assert_allclose(out.numpy(), g["ddpm"], rtol=1e-4, atol=1e-4)


def test_canonical_target():
    tg = b200mdm.synthetic_target_inputs(5, seed=2)
    tc, valid = canonical_target(tg, 5, JOINTS)
    assert tc is tg["target_cond"] and valid.dtype == np.uint8
    np.testing.assert_array_equal(valid, to.validity(JOINTS, tg["target_joint_names"], tg["is_heading"]).numpy())
    assert valid[0, JOINTS.index("heading")] == 1 and valid[1, JOINTS.index("heading")] == 0
    # plain lists of names, heading as a list
    y = dict(target_cond=tg["target_cond"][:2], target_joint_names=[["pelvis"], []], is_heading=[False, True])
    _, v = canonical_target(y, 2, JOINTS)
    assert v.sum() == 2 and v[0, 0] == 1 and v[1, -1] == 1
    y["target_joint_names"] = [["pelvis"], ["left_knee"]]
    with pytest.raises(ValueError, match="left_knee"):
        canonical_target(y, 2, JOINTS)
    with pytest.raises(ValueError):
        canonical_target(dict(y, target_cond=torch.zeros(2, 7, 3)), 2, JOINTS)


def test_shard_slices_target_keys():
    tg = b200mdm.synthetic_target_inputs(6, seed=3)
    y = dict(tg, scale=torch.ones(6))
    out = shard_model_kwargs({"y": y}, 2, 5)["y"]
    assert torch.equal(out["target_cond"], tg["target_cond"][2:5])
    assert torch.equal(out["is_heading"], tg["is_heading"][2:5])
    assert [list(n) for n in out["target_joint_names"]] == [list(n) for n in tg["target_joint_names"][2:5]]
    y = dict(target_cond=tg["target_cond"].numpy(), is_heading=tg["is_heading"].numpy(),
             target_joint_names=np.array(tg["target_joint_names"], dtype=object))
    out = shard_model_kwargs({"y": y}, 1, 3)["y"]
    assert out["target_cond"].shape == (2, 8, 3) and out["is_heading"].shape == (2,) and len(out["target_joint_names"]) == 2


def test_autoregressive_sampler_passes_target_to_every_chunk():
    tg = b200mdm.synthetic_target_inputs(2, seed=4)
    seen = []

    def sample_fn(model, shape, **kw):
        seen.append(kw["model_kwargs"]["y"])
        return torch.zeros(shape)
    args = SimpleNamespace(pred_len=40, context_len=20)
    y = dict(tg, prefix=torch.zeros(2, 263, 1, 20))
    b200mdm.AutoRegressiveSampler(args, sample_fn, required_frames=100).sample(None, (2, 263, 1, 40), model_kwargs={"y": y})
    assert len(seen) == 3
    for yc in seen:
        assert all(yc[k] is tg[k] for k in tg)
