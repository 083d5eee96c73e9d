"""Cases of the guided DDPM / DDIM step (tests/test_guided_step_gpu.py, tests/test_guided_step_cpu.py): a model, one x_t
with its noise, the joint, foot and scene guidance inputs, the tail's flags, and the wiring mutants each case can see.

Everything is built on the host from seeds, so both files see the same inputs: the GPU file takes the step's x0 from
the engine, the CPU file from the fp32 oracle denoiser.  The guidance inputs of one motion are its rows of the
per-sample tensors; a mutant re-reads them through another index map or drops one term, as a wiring mistake in the
engine would (DESIGN.md, "Joint-position control", "The guided step")."""
from types import SimpleNamespace

import torch

import b200mdm
from conftest import default_args
from oracle import dec_emb_oracle as deo
from oracle import foot_guidance_oracle as fo
from oracle import joint_control_oracle as jo
from oracle import mdm_oracle as mo
from oracle import plms_oracle as po
from oracle import ric_oracle
from oracle import scene_guidance_oracle as so

U32 = 2.0 ** -24
EPS_G = 2.0 ** -12          # relative error of the kernel's guidance displacement (DESIGN.md)
EPS_L = 2.0 ** -16          # relative error of its per-iteration loss
MISS = 8.0                  # every mutant misses the bound by at least this factor
CW, FW, FH, OW, R = 4.0, 2.0, 0.0, 4.0, 0.3
PREV = (0.5, 5)             # the "previous upload" of the lambda / K mutant: lambda * 0.5, K = 5

# name: arch, layers, steps, B, T, lengths, scales, features, [(sampler, eta, schedule index)], clip, inpainting and
# jw, the joint weights' scale (it balances the joint term against the foot and scene terms, so each mutant shows)
CASES = {
    "enc_joint": dict(arch="enc", L=2, steps=6, B=4, T=40, lengths=[40, 31, 17, 9], scales=[0.0, 1.0, 2.5, 7.5],
                      feat="joint", steps_run=[("ddpm", 0.0, 5), ("ddim", 0.0, 3)], clip=False, inpaint=None),
    "enc_joint_foot": dict(arch="enc", L=2, steps=6, B=4, T=40, lengths=[40, 31, 17, 9], scales=[0.0, 1.0, 2.5, 7.5],
                           feat="joint_foot", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.5, 0)], clip=True, inpaint="bool"),
    "enc_foot_given": dict(arch="enc", L=2, steps=6, B=3, T=40, lengths=[40, 28, 13], scales=[2.5, 1.0, 7.5],
                           feat="foot_given", steps_run=[("ddpm", 0.0, 0), ("ddim", 0.0, 5)], clip=False, inpaint="soft"),
    "enc_scene_sdf_shared": dict(arch="enc", L=2, steps=6, B=3, T=40, lengths=[40, 22, 11], scales=[2.5, 2.5, 7.5],
                                 feat="scene_shared_sdf", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.5, 5)], clip=True,
                                 inpaint=None, jw=20.0),
    "enc_scene_sdf_per_sample": dict(arch="enc", L=2, steps=6, B=3, T=40, lengths=[40, 31, 17], scales=[2.5, 0.0, 7.5],
                                     feat="scene_ps_sdf", steps_run=[("ddpm", 0.0, 5), ("ddim", 0.0, 0)], clip=False,
                                     inpaint="bool", jw=20.0),
    "kit_joint_foot": dict(arch="kit", L=2, steps=6, B=3, T=48, lengths=[48, 35, 20], scales=[2.5, 7.5, 1.0],
                           feat="joint_foot", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.0, 5)], clip=False, inpaint=None),
    "clip_dec_joint_foot": dict(arch="clip", L=2, steps=6, B=3, T=40, lengths=[40, 33, 20], scales=[2.5, 7.5, 0.0],
                                feat="joint_foot", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.5, 3)], clip=False,
                                inpaint=None),
    "bert_dec_t256_joint": dict(arch="bert", L=2, steps=6, B=2, T=256, lengths=[256, 190], scales=[2.5, 7.5],
                                feat="joint", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.0, 5)], clip=False, inpaint=None),
    "enc_t1_joint_foot": dict(arch="enc", L=2, steps=6, B=3, T=1, lengths=[1, 1, 1], scales=[2.5, 7.5, 1.0],
                              feat="joint_foot", steps_run=[("ddpm", 0.0, 3), ("ddim", 0.0, 0)], clip=False, inpaint=None),
    "enc_t2_scene": dict(arch="enc", L=2, steps=6, B=3, T=2, lengths=[2, 1, 2], scales=[2.5, 7.5, 1.0],
                         feat="scene_ps_sdf", steps_run=[("ddpm", 0.0, 5), ("ddim", 0.5, 3)], clip=False, inpaint=None),
}
HEADLINE = {   # one step per feature set at the headline shape; the fp64 parts follow three of the 64 motions
    "head_joint": dict(arch="enc", L=8, steps=50, B=64, T=196, lengths=None, scales=[2.5], feat="joint",
                       steps_run=[("ddpm", 0.0, 25)], clip=False, inpaint=None, idx=[0, 31, 63]),
    "head_joint_foot": dict(arch="enc", L=8, steps=50, B=64, T=196, lengths="ragged", scales=[2.5], feat="joint_foot",
                            steps_run=[("ddpm", 0.0, 25)], clip=False, inpaint=None, idx=[0, 31, 63], jw=0.05),
    "head_scene": dict(arch="enc", L=8, steps=50, B=64, T=196, lengths="ragged", scales=[2.5], feat="scene_ps_sdf",
                       steps_run=[("ddpm", 0.0, 25)], clip=False, inpaint=None, idx=[0, 31, 63], jw=20.0),
}


def feats(arch):
    return 251 if arch == "kit" else 263


def model_args(c):
    """(args of create_model_and_diffusion, synthetic_state_dict kwargs)"""
    L, steps = c["L"], c["steps"]
    if c["arch"] == "kit":
        return default_args(dataset="kit", layers=L, diffusion_steps=steps), dict(num_layers=L, input_feats=251, seed=81)
    if c["arch"] == "clip":
        return (default_args(layers=L, diffusion_steps=steps, arch="trans_dec", emb_trans_dec=True),
                dict(arch="trans_dec", num_layers=L, cond_dim=512, seed=0))
    if c["arch"] == "bert":
        return (default_args(layers=L, diffusion_steps=steps, arch="trans_dec", text_encoder_type="bert"),
                dict(arch="trans_dec", num_layers=L, cond_dim=768, seed=0))
    return default_args(layers=L, diffusion_steps=steps), dict(num_layers=L, seed=1)


def _planar(B, slopes, o=(-2.0, -1.5), c=0.25, gz=12, gx=14):
    z = o[1] + c * torch.arange(gz, dtype=torch.float64)
    x = o[0] + c * torch.arange(gx, dtype=torch.float64)
    return b200mdm.SceneGrid(torch.stack([a + sx * x[None, :] + sz * z[:, None] for a, sx, sz in slopes[:B]]), o, c)


def _grids(feat, B, g):
    """(obstacle sdf, terrain): planar grids (their bilinear gradient is continuous, so fp32 and fp64 pick equivalent
    cells) per sample or shared, or a curved SDF of discs and a box shared by the batch"""
    sl = [(0.3 + 0.1 * float(torch.rand(1, generator=g)), 0.8 - 0.2 * b, -0.5 + 0.3 * b) for b in range(B)]
    tl = [(0.05 - 0.02 * b, 0.3 - 0.1 * b, 0.2 + 0.05 * b) for b in range(B)]
    if feat == "scene_ps_sdf":
        ter = _planar(1, tl)
        return _planar(B, sl), b200mdm.SceneGrid(ter.values[0], ter.origin, ter.cell)
    sdf = b200mdm.SceneGrid.from_shapes((17, 17), (-2.0, -2.0), 0.25, discs=[(0.0, 0.0, 0.4), (0.8, -0.6, 0.3)],
                                        boxes=[(-1.2, 0.5, -0.4, 0.8)])
    return sdf, _planar(B, tl)


def _positions(x, mean, std):
    D = x.shape[1]
    data = (x.double() * std.double()[None, :, None] + mean.double()[None, :, None]).permute(0, 2, 1)
    return ric_oracle.recover_from_ric(data, jo.n_joints(D)).permute(0, 2, 3, 1)   # [B, J, 3, T]


def build(c, seed=1):
    """The host inputs of case c: SimpleNamespace of every tensor and weight both files use (fp32, CPU)."""
    g = torch.Generator().manual_seed(seed)
    B, T, D = c["B"], c["T"], feats(c["arch"])
    J = jo.n_joints(D)
    mean, std = jo.motion_stats(D)
    lengths = c["lengths"]
    if lengths is None:
        lengths = [T] * B
    elif lengths == "ragged":
        lengths = [T - (37 * b) % (T // 2) for b in range(B)]
    scales = c["scales"] * (B // len(c["scales"])) if len(c["scales"]) < B else c["scales"]
    inp = b200mdm.synthetic_inputs(B, njoints=D, nframes=T, steps=c["steps"], seed=seed + 10, lengths=lengths,
                                   scale=torch.tensor(scales, dtype=torch.float32))
    text = None
    if c["arch"] == "bert":
        enc, tmask, _ = b200mdm.synthetic_dip_inputs(B, 20, 0, seed=13)
        text = (enc, tmask)
    xt = torch.randn(B, D, 1, T, generator=g)
    noise = torch.randn(B, D, 1, T, generator=g)
    feat = c["feat"]
    target = _positions(torch.randn(B, D, T, generator=g) * 0.5, mean, std).float()
    weight = torch.zeros(B, J, T)
    if feat != "foot_given":
        weight[:, 0] = 1.0                                            # the pelvis on every frame
        for j in (20, 21) if J == 22 else (4, 7):                     # the wrists at sparse keyframes
            weight[:, j, torch.arange(T // 5, T, max(1, T // 4))] = 1.0
        weight *= c.get("jw", 1.0)
    foot = feat != "joint"
    contact = None
    if feat == "foot_given":
        contact = torch.rand(B, 4, T, generator=g) * 1.5 * (torch.rand(B, 4, T, generator=g) < 0.6)
    sdf = terrain = None
    if feat.startswith("scene"):
        sdf, terrain = _grids(feat, B, g)
    extent = float(target[:, :, [0, 2]].max() - target[:, :, [0, 2]].min()) + 2.0
    kmax = 1.0 if contact is None else float(contact.max())
    cw, fw = (CW, FW) if foot else (0.0, 0.0)
    if sdf is not None:
        # so.step_bound's grid terms (2 lo s_S^2 J T g) leave lambda too small to move x0 past the bound's rounding
        # floor; the scene terms are taken as one more floor-like term of unit slope instead (the hook's error against
        # fp64 is measured at this lambda)
        step = fo.step_bound(std, weight, extent, T, cw, fw + OW, kmax)
    elif foot:
        step = fo.step_bound(std, weight, extent, T, cw, fw, kmax)
    else:
        step = jo.step_bound(std, weight, extent, T)
    mask = soft = motion = None
    if c["inpaint"] is not None:
        motion = torch.randn(B, D, 1, T, generator=g) * 0.5
        if c["inpaint"] == "bool":
            mask = torch.rand(B, D, 1, T, generator=g) < 0.2
            mask[..., : max(1, T // 8)] = True
        else:
            soft = torch.rand(B, D, 1, T, generator=g)
            soft[soft < 0.2] = 0.0
            soft[soft > 0.9] = 1.0
    idx = c.get("idx", list(range(B)))
    return SimpleNamespace(c=c, B=B, T=T, D=D, J=J, mean=mean, std=std, inp=inp, text=text, xt=xt, noise=noise,
                           target=target, weight=weight, joint=feat != "foot_given", foot=foot, contact=contact,
                           lengths=inp["lengths"], scale=inp["scale"], sdf=sdf, terrain=terrain, cw=cw, fw=fw, fh=FH,
                           ow=OW if sdf is not None else 0.0, r=R, step=step, iters=10, clip=c["clip"], mask=mask,
                           soft=soft, motion=motion, idx=idx)


def y_dict(k, device, scale=None, **extra):
    """y of the case: conditioning, guidance keys and inpainting, on `device`"""
    inp = k.inp
    y = dict(mask=inp["mask"].to(device), lengths=inp["lengths"].to(device),
             text_embed=(tuple(t.to(device) for t in k.text) if k.text is not None else inp["text_embed"].to(device)),
             scale=(inp["scale"] if scale is None else scale).to(device))
    if k.joint:
        y.update(joint_target=k.target.to(device), joint_weight=k.weight.to(device))
    if k.contact is not None:
        y["foot_contact"] = k.contact.to(device)
    if k.sdf is not None:
        y.update(obstacle_sdf=k.sdf, terrain=k.terrain)
    if k.mask is not None:
        y.update(inpainting_mask=k.mask.to(device), inpainted_motion=k.motion.to(device))
    if k.soft is not None:
        y.update(inpainting_weight=k.soft.to(device), inpainted_motion=k.motion.to(device))
    y.update(extra)
    return y


def wrapper_kw(k):
    """JointControlSampleModel keywords of the case"""
    kw = {}
    if k.foot:
        kw.update(contact_weight=k.cw, floor_weight=k.fw, floor_height=k.fh)
    if k.sdf is not None:
        kw.update(obstacle_weight=k.ow, obstacle_margin=k.r)
    return kw


# ------------------------------------------------------------------------------------------------ guidance inputs
def _rows(v, rows):
    return None if v is None else v[rows]


def _grid_rows(grid, rows):
    return grid if grid is None or not grid.per_sample else b200mdm.SceneGrid(grid.values[rows], grid.origin, grid.cell)


def guide_inputs(k, rows=None):
    """the guidance inputs of motions `rows` (default k.idx): a dict of the oracles' and hooks' keyword arguments"""
    rows = k.idx if rows is None else rows
    return dict(target=k.target[rows], weight=k.weight[rows], contact=_rows(k.contact, rows),
                lengths=k.lengths[rows], sdf=_grid_rows(k.sdf, rows), terrain=_grid_rows(k.terrain, rows),
                step=k.step, iters=k.iters, foot=k.foot, scene=k.sdf is not None)


def mutants(k, rows=None):
    """{name: (guidance inputs, x0 source, tail order)} of the wiring mistakes case k can see, for motions `rows`
    (default k.idx).  x0 source: "raw" (the step's CFG x0) or "cond" (the conditional x0, scale 1); tail order: None
    (guidance, then inpainting, then the clamp), "after_inpaint" or "after_clamp"."""
    idx, B, T = (k.idx if rows is None else rows), k.B, k.T
    nxt = [(b + 1) % B for b in idx]
    base = guide_inputs(k, idx)
    m = {}
    if k.joint:
        m["targets_next"] = (dict(target=k.target[nxt], weight=k.weight[nxt]), "raw", None)
    if any(float(k.scale[b]) != 1.0 for b in idx):
        m["cond_x0"] = ({}, "cond", None)
    if k.foot or k.sdf is not None:
        if any(int(k.lengths[b]) < T for b in idx):
            m["no_lengths"] = (dict(lengths=None), "raw", None)
        if not torch.equal(k.lengths[nxt], k.lengths[idx]):
            m["lengths_next"] = (dict(lengths=k.lengths[nxt]), "raw", None)
    if k.contact is not None:
        m["contact_next"] = (dict(contact=k.contact[nxt]), "raw", None)
    for name, grid in (("sdf", k.sdf), ("terrain", k.terrain)):
        if grid is not None and grid.per_sample:
            m["%s_next" % name] = ({name: _grid_rows(grid, nxt)}, "raw", None)
            m["%s_of_sample_0" % name] = ({name: b200mdm.SceneGrid(grid.values[0], grid.origin, grid.cell)}, "raw", None)
    m["prev_upload"] = (dict(step=k.step * PREV[0], iters=PREV[1]), "raw", None)
    if k.foot and k.sdf is None:
        m["no_foot"] = (dict(foot=False), "raw", None)
    if k.sdf is not None:
        m["no_scene"] = (dict(scene=False), "raw", None)
    if k.mask is not None or k.soft is not None:
        m["after_inpaint"] = ({}, "raw", "after_inpaint")
    if k.clip:
        m["after_clamp"] = ({}, "raw", "after_clamp")
    return {name: (dict(base, **chg), src, order) for name, (chg, src, order) in m.items()}


def guide64(k, x0, g):
    """(guided x0 fp64 [n, D, T], loss fp64 [K + 1, n]) of normalised x0 [n, D, T] by the fp64 oracle of the terms g
    switches on"""
    x0 = x0.reshape(x0.shape[0], x0.shape[1], x0.shape[-1])
    if g["scene"]:
        return so.guide(x0, k.mean, k.std, g["target"], g["weight"], g["step"], g["iters"], k.cw, k.fw, k.fh, k.ow, k.r,
                        g["sdf"], g["terrain"], g["contact"], g["lengths"])
    if g["foot"]:
        return fo.guide(x0, k.mean, k.std, g["target"], g["weight"], g["step"], g["iters"], k.cw, k.fw, k.fh,
                        g["contact"], g["lengths"])
    return jo.guide(x0, k.mean, k.std, g["target"], g["weight"], g["step"], g["iters"])


def inpaint(k, x, rows, f64=False):
    """the inpainting of motions `rows` of x [n, D, T]: the bool mask's select or the soft blend (fp32 with every op
    rounded, as soft_inpaint; fp64 with f64)"""
    if k.mask is None and k.soft is None:
        return x
    shp = x.shape
    mo_ = k.motion[rows].reshape(shp).to(x.device, x.dtype)
    if k.mask is not None:
        return torch.where(k.mask[rows].reshape(shp).to(x.device), mo_, x)
    w = k.soft[rows].reshape(shp).to(x.device, x.dtype)
    a = (1 - w) * x
    b = w * mo_
    blend = a + b
    return torch.where(w >= 1, mo_, torch.where(w <= 0, x, blend))


def clamp(k, x):
    return x.clamp(-1, 1) if k.clip else x


def bound(k, x0, want, iters):
    """the fp64 bound of DESIGN.md: 2^-12 max |guided - x0| + 2 u K max |x0|"""
    x0 = x0.reshape(want.shape).double()
    return EPS_G * float((want - x0).abs().max()) + 2 * U32 * iters * float(x0.abs().max())


# ------------------------------------------------------------------------------------------------ the fp32 oracle x0
def oracle_denoiser(k, sd, rows, scale=None):
    """denoise(x, i) -> x0 [n, D, 1, T] fp32 of the case's model for motions `rows` (the CFG blend at k's scales, or at
    `scale`)"""
    c = k.c
    W = mo.OracleWeights(sd, c["L"])
    sc = (k.scale if scale is None else scale)[rows]
    te, ln = k.inp["text_embed"][:, rows], k.lengths[rows]
    if c["arch"] == "bert":
        enc, tmask = k.text[0][:, rows], k.text[1][rows]
        return lambda x, i: mo.cfg_denoise_dec(W, x, i, enc, tmask, x.new_zeros(x.shape[:-1] + (0,)), sc, ln)
    if c["arch"] == "clip":
        return deo.denoiser(W, list(range(c["steps"])), te, sc, ln)
    return po.enc_denoiser(W, list(range(c["steps"])), te, sc, ln)
