"""GPU: goal-directed autoregressive chains (AutoRegressiveSampler with y['target_world']; DESIGN.md, "Goals in the
world frame").

  * b200mdm_chunk_frame, chunk by chunk over the reference fixture, against the reference's chunk-local targets and
    the fp64 oracle's carry;
  * the device chain bit for bit equal to the host chain (which runs the same kernel), across samplers, include_prefix,
    one goal and per-chunk goals, a crop inside the last chunk, and the single and multi target encoders;
  * the device chain against an fp32 oracle chain whose chunk targets come from oracle/goal_oracle.py;
  * chunk 0 without a prefix equal to the static-target chain's; batch halves equal to the whole batch;
  * exactly two more launches per chunk boundary, and b200mdm_chain_set_goal's own apart."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import b200mdm
from b200mdm import parallel
from b200mdm.engine import Engine
from conftest import default_args, rel_err
from oracle import goal_oracle as go
from oracle import mdm_oracle as mo
from oracle import schedule_oracle as so
from oracle import target_oracle as to
import test_ar_chain_gpu as ac

pytestmark = pytest.mark.gpu
L, CTX, PRED, STEPS, C = ac.L, ac.CTX, ac.PRED, ac.STEPS, ac.C
EXT = ["pelvis", "left_foot", "right_foot", "left_wrist", "right_wrist", "head", "traj", "heading"]


def build(encoder="multi", seed=21):
    over = dict(layers=L, diffusion_steps=STEPS, arch="trans_dec", text_encoder_type="bert", context_len=CTX,
                pred_len=PRED, multi_target_cond=True, multi_encoder_type=encoder, target_enc_layers=1)
    model, diffusion = b200mdm.create_model_and_diffusion(default_args(**over), SimpleNamespace(dataset=SimpleNamespace()))
    sd = b200mdm.synthetic_state_dict(arch="trans_dec", num_layers=L, cond_dim=C, seed=seed, target_encoder=encoder)
    b200mdm.load_model_wo_clip(model, sd)
    model.to("cuda").eval()
    model.clip_model = ac.FakeBert(6)
    return model, diffusion, sd


def norm_stats():
    g = torch.Generator().manual_seed(17)
    return (torch.randn(263, generator=g) * 0.1).cuda(), (0.5 + torch.rand(263, generator=g)).cuda()


def goal_y(B, n_chunks, per_chunk, seed=3):
    y = ac.make_y(B, n_chunks, seed=seed)
    tg = b200mdm.synthetic_target_inputs(B, seed=5)
    g = torch.Generator().manual_seed(seed + 40)
    shape = (n_chunks, B, len(EXT), 3) if per_chunk else (B, len(EXT), 3)
    goal = torch.randn(shape, generator=g) * 2.0
    goal[..., EXT.index("traj"), 1] = 0.0
    goal[..., EXT.index("heading"), 0] = torch.rand(shape[:-2], generator=g) * 2 * math.pi - math.pi
    y.update(target_world=goal.cuda(), target_joint_names=tg["target_joint_names"], is_heading=tg["is_heading"])
    return y


def sample(model, diffusion, sampler, y, required, include_prefix, host=False, seed=5, B=3, **kw):
    args = SimpleNamespace(pred_len=PRED, context_len=CTX, autoregressive_include_prefix=include_prefix)
    fn = getattr(diffusion, sampler)
    mean, std = norm_stats()
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    s = b200mdm.AutoRegressiveSampler(args, ac.host(fn) if host else fn, required_frames=required, mean=mean, std=std)
    kw = dict(kw)
    if sampler != "dpm_solver_sample_loop":
        kw.setdefault("clip_denoised", False)
    out = s.sample(b200mdm.ClassifierFreeSampleModel(model), (B, 263, 1, PRED), model_kwargs={"y": y}, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", ["prefix", "noprefix"])
def test_chunk_frame_against_golden_and_oracle(golden, case):
    z = golden("goal_frames.npz")
    off = int(z["ctx"]) if case == "prefix" else 0
    pred, n = int(z["pred"]), int(z["n_chunks"])
    mean, std, motion = (torch.from_numpy(z[k]) for k in ("mean", "std", case + "_motion"))
    names = [[j for j in str(s).split(";") if j] for s in z["names"]]
    B = motion.shape[0]
    carry = torch.zeros(B, 6, dtype=torch.float64, device="cuda")
    md = motion.cuda()
    for c in range(n):
        lo, hi = (0, off) if c == 0 else (off + (c - 1) * pred, off + c * pred)
        world = torch.from_numpy(z["%s_world_%d" % (case, c)])
        local = torch.from_numpy(z["%s_local_%d" % (case, c)]).double()
        got = Engine.chunk_frame(carry, md[..., lo:hi], mean.cuda(), std.cuda(), world.cuda()).cpu().double()
        torch.cuda.synchronize()
        ref_carry = go.carry_after(motion, mean, std, hi)
        assert float((carry.cpu() - ref_carry).abs().max()) < 1e-6, c
        oracle = go.to_chunk(world, go.frame_at(motion, mean, std, hi))
        for b in range(B):
            for j in names[b]:
                i = EXT.index(j)
                assert float((got[b, i] - local[b, i]).norm() / local[b, i].norm()) < 1e-5, (c, b, j)
                assert float((got[b, i] - oracle[b, i]).norm() / oracle[b, i].norm()) < 1e-6, (c, b, j)
            if z["is_heading"][b]:
                d = float(got[b, -1, 0] - local[b, -1, 0])
                assert abs((d + math.pi) % (2 * math.pi) - math.pi) < 1e-5, (c, b)
        if c == 0 and off == 0:
            assert torch.equal(got.float(), world)


CASES = {
    # name: (sampler, sampler kwargs, include_prefix, per-chunk goals, required frames, encoder)
    "ddpm_prefix_one": ("p_sample_loop", {}, True, False, 32, "multi"),
    "ddpm_noprefix_waypoints_crop": ("p_sample_loop", {}, False, True, 29, "multi"),
    "ddim_prefix_waypoints": ("ddim_sample_loop", {"eta": 0.5}, True, True, 32, "multi"),
    "ddim_noprefix_one_single": ("ddim_sample_loop", {"eta": 0.0}, False, False, 30, "single"),
    "dpm2_prefix_one_crop": ("dpm_solver_sample_loop", {"order": 2}, True, False, 27, "multi"),
    "dpm2_noprefix_waypoints_single": ("dpm_solver_sample_loop", {"order": 2}, False, True, 32, "single"),
}


@pytest.fixture(scope="module")
def models():
    return {enc: build(enc) for enc in ("multi", "single")}


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_chain_equals_host_chain(models, case):
    sampler, skw, include_prefix, per_chunk, required, enc = CASES[case]
    model, diffusion, _ = models[enc]
    n_chunks = -(-required // PRED)
    y = goal_y(3, n_chunks, per_chunk)
    dev = sample(model, diffusion, sampler, y, required, include_prefix, **skw)
    hst = sample(model, diffusion, sampler, y, required, include_prefix, host=True, **skw)
    assert dev.shape == (3, 263, 1, required)
    assert torch.equal(dev, hst), float((dev - hst).abs().max())
    # the goal changes the chain: the same chain with the goal as a static target differs after chunk 0
    static = dict(y, target_cond=y["target_world"][0] if per_chunk else y["target_world"])
    del static["target_world"]
    other = sample(model, diffusion, sampler, static, required, include_prefix, **skw)
    off = CTX if include_prefix else 0
    assert not torch.equal(dev[..., off + PRED:], other[..., off + PRED:])


def test_identity_chunk_without_prefix(models):
    model, diffusion, _ = models["multi"]
    y = goal_y(3, 3, False)
    dev = sample(model, diffusion, "p_sample_loop", y, 24, False)
    static = dict(y, target_cond=y["target_world"])
    del static["target_world"]
    ref = sample(model, diffusion, "p_sample_loop", static, 24, False)
    assert torch.equal(dev[..., :PRED], ref[..., :PRED])


def test_device_chain_against_fp32_oracle(models):
    model, diffusion, sd = models["multi"]
    B, required = 3, 24
    n_chunks = required // PRED
    shape = (B, 263, 1, PRED)
    y = goal_y(B, n_chunks, True)
    nk = ac.noise_kw("tape", n_chunks, STEPS, shape)
    out = sample(model, diffusion, "p_sample_loop", y, required, True, **nk)
    mean, std = (t.cpu() for t in norm_stats())
    W = mo.OracleWeights(sd, L, arch="trans_dec")
    tabs = so.diffusion_tables(so.named_betas("cosine", STEPS))
    enc, tmask = y["text_embed"][0].cpu(), y["text_embed"][1].cpu()
    valid = to.validity(EXT, y["target_joint_names"], y["is_heading"])
    goals = y["target_world"].cpu()
    prefix, returned = y["prefix"].cpu(), [y["prefix"].cpu()]
    for c in range(n_chunks):
        motion = torch.cat(returned, -1)
        fr = go.frame_at(motion, mean, std, CTX + c * PRED)
        tgt = go.to_chunk(goals[c], fr).float()
        g = to.target_embedding(W, "multi", tgt, valid, joint_names=EXT)
        tape = [nk["noise"][c].cpu()] + list(nk["noise_tape"][c].cpu())
        x = to.sample_loop_dec(W, tabs, list(range(STEPS)), tape, enc, tmask, prefix, g, y["scale"].cpu(), y["lengths"].cpu())
        returned.append(x)
        prefix = x[..., -CTX:]
    ref = torch.cat(returned, -1)[..., :required]
    assert rel_err(out, ref) < 1e-3


def test_batch_halves_equal_whole_batch(models):
    model, diffusion, _ = models["multi"]
    B = 4
    y = goal_y(B, 4, True)
    whole = sample(model, diffusion, "p_sample_loop", y, 30, True, B=B, noise_seed=77)
    halves = []
    for lo, hi in ((0, 2), (2, 4)):
        yh = parallel.shard_model_kwargs({"y": y}, lo, hi)["y"]
        halves.append(sample(model, diffusion, "p_sample_loop", yh, 30, True, B=2, noise_seed=77, sample_index_base=lo))
    assert torch.equal(whole, torch.cat(halves))


@pytest.mark.parametrize("use_graph", [True, False])
def test_launch_count(models, monkeypatch, use_graph):
    model, diffusion, _ = models["multi"]
    eng = model.engine()
    counts = {}
    orig_loop, orig_goal = Engine.chain_loop_range, Engine.chain_set_goal

    def counted(orig, key):
        def f(self, *a, **k):
            torch.cuda.synchronize()
            before = self.launch_count()
            r = orig(self, *a, **k)
            counts[key] = counts.get(key, 0) + self.launch_count() - before
            return r
        return f
    n_chunks = 4
    y = goal_y(3, n_chunks, True)
    static = dict(y, target_cond=y["target_world"][0])
    del static["target_world"]
    res = {}
    for name, yy in (("goal", y), ("static", static)):
        for _ in range(2):                           # the second run: graphs captured
            counts.clear()
            monkeypatch.setattr(Engine, "chain_loop_range", counted(orig_loop, "loop"))
            monkeypatch.setattr(Engine, "chain_set_goal", counted(orig_goal, "goal"))
            sample(model, diffusion, "p_sample_loop", yy, 32, True, use_graph=use_graph, noise_seed=3)
        res[name] = dict(counts)
    assert eng is model.engine()
    assert res["goal"]["loop"] == res["static"]["loop"] + 2 * (n_chunks - 1)
    assert res["goal"]["goal"] == 2 and "goal" not in res["static"]
