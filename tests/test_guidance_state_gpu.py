"""GPU: which terms of joint-position control stay live across setter calls, checked against a fresh engine bit for bit.

Each setter of b200mdm_set_{joint,foot,scene,interaction}_guidance clears its own term and the terms above it, and
b200mdm_set_cond* clears them all; a foot call with both weights 0 keeps its lengths for the scene terms.  Each sequence
below runs on one long-lived engine (the reused engine, which carries the state of the sequences before it), then one
DDPM loop through the step graph and one with plain launches.  A fresh engine given only the terms that should still be
live runs the same two loops: the samples must have the same bits and the loops the same launch count."""
import pytest
import torch

import b200mdm
from b200mdm import _lib
from b200mdm.engine import Engine
from b200mdm.utils.model_util import create_gaussian_diffusion
from b200mdm.utils.scene import SceneGrid
from conftest import default_args
from oracle import schedule_oracle as so

pytestmark = pytest.mark.gpu
L, STEPS, B, T, C, J = 2, 6, 4, 24, 2, 22
CFG = dict(arch="trans_enc", latent_dim=512, ff_size=1024, num_layers=L, num_heads=4, njoints=263, nfeats=1,
           cond_mode="text", cond_dim=512, num_actions=1, mask_frames=True, pos_embed_max_len=5000, temb_rows=1000)
ITERS, FH, OW, R, LA, RA = 4, -0.2, 4.0, 0.2, 4.0, 0.3


def same(a, b):
    """The same bits (NaN payloads and signed zeros included)."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().reshape(-1).view(torch.uint8),
                                                                     b.contiguous().reshape(-1).view(torch.uint8))


class Inputs:
    """Weights, schedule, conditioning, noise and two argument sets of every term, from one seed."""

    def __init__(self, seed=71):
        g = torch.Generator().manual_seed(seed)
        self.sd = b200mdm.synthetic_state_dict(num_layers=L, seed=61)
        self.sd["sequence_pos_encoder.pe"] = so.positional_table(CFG["pos_embed_max_len"], 512)
        d = create_gaussian_diffusion(default_args(layers=L, diffusion_steps=STEPS))
        self.rows, self.tmap = d.schedule_rows(0.0), list(range(STEPS))
        lengths = torch.tensor([T, 17, 9, T], dtype=torch.int64)
        self.y = dict(lengths=lengths.cuda(), text_embed=torch.randn(1, B, 512, generator=g).cuda(),
                      scale=torch.tensor([2.5, 1.0, 0.0, 2.0]).cuda())
        self.lengths = lengths
        mean, std = b200mdm.synthetic_norm_stats(263)
        self.mean, self.std = mean.cuda(), std.cuda()
        self.target = [(torch.randn(B, J, 3, T, generator=g) * 0.5).cuda() for _ in range(2)]
        self.weight = [(torch.rand(B, J, T, generator=g) < 0.3).float().cuda() for _ in range(2)]
        self.step = [2e-5, 4e-5]
        self.sdf = SceneGrid(torch.rand(8, 8, generator=g) * 0.4 - 0.1, (-2.0, -2.0), 0.5)
        self.terrain = SceneGrid(torch.rand(B, 8, 8, generator=g) * 0.05, (-2.0, -2.0), 0.5)
        self.placement = torch.tensor([[0.0, 0.0, 0.0], [0.3, 0.1, 1.0], [0.0, 0.0, -0.5], [0.2, -0.2, 2.0]]).cuda()
        self.pairs = torch.tensor([[0, 20, 1, 21], [1, 15, 0, 10]], dtype=torch.int32)
        self.reach = torch.tensor([0.1, 0.4])
        self.pair_weight = torch.rand(2, T, generator=g).cuda()
        shape = (B, 263, 1, T)
        self.x = torch.randn(shape, generator=g).cuda()
        self.tape = torch.randn((STEPS,) + shape, generator=g).cuda()

    def engine(self):
        eng = Engine(**CFG)
        eng.load_state_dict(self.sd)
        eng.set_schedule(self.rows, self.tmap)
        self.set_cond(eng)
        return eng

    def set_cond(self, eng):
        eng.set_cond(B, T, self.y, True, torch.device("cuda"))

    # the terms; v picks one of two argument sets
    def joint(self, eng, v=0):
        eng.set_joint_guidance(self.mean, self.std, self.target[v], self.weight[v], self.step[v], ITERS)

    def foot(self, eng, contact_weight, floor_weight):
        eng.set_foot_guidance(contact_weight, floor_weight, FH, None, self.lengths)

    def scene(self, eng, terrain):
        eng.set_scene_guidance(OW, R, self.sdf, self.terrain if terrain else None)

    def interaction(self, eng):
        eng.set_interaction_guidance(C, LA, RA, self.placement, self.pairs, self.reach, self.pair_weight)

    def loops(self, eng):
        """(samples, launch count) of a DDPM loop through the step graph, then of one with plain launches"""
        out = []
        for use_graph in (True, False):
            torch.cuda.synchronize()
            eng.launch_count(reset=True)
            x0 = eng.sample_loop(_lib.MODE_DDPM, self.x, self.tape, use_graph=use_graph)
            torch.cuda.synchronize()
            out.append((x0, eng.launch_count()))
        return out


# (name, the calls on the reused engine, the calls on a fresh engine that leave the same terms live)
SEQUENCES = [
    ("joint, foot, scene, interaction, then foot again",
     lambda i, e: (i.joint(e), i.foot(e, 4.0, 2.0), i.scene(e, True), i.interaction(e), i.foot(e, 1.0, 3.0)),
     lambda i, e: (i.joint(e), i.foot(e, 1.0, 3.0))),
    ("joint, scene without foot, then joint again",
     lambda i, e: (i.joint(e, 1), i.scene(e, False), i.joint(e)),
     lambda i, e: i.joint(e)),
    ("foot with both weights 0, then scene (the lengths kept, the foot terms off)",
     lambda i, e: (i.foot(e, 0.0, 0.0), i.scene(e, False)),
     lambda i, e: (i.joint(e), i.foot(e, 0.0, 0.0), i.scene(e, False))),
    ("interaction, set_cond, then joint",
     lambda i, e: (i.joint(e, 1), i.interaction(e), i.set_cond(e), i.joint(e)),
     lambda i, e: i.joint(e)),
]


def test_setter_sequences_against_fresh_engine():
    inp = Inputs()
    eng = inp.engine()
    try:
        for name, reused_calls, fresh_calls in SEQUENCES:
            reused_calls(inp, eng)
            got = inp.loops(eng)
            fresh = inp.engine()
            try:
                fresh_calls(inp, fresh)
                want = inp.loops(fresh)
            finally:
                fresh.close()
            for (g, gn), (w, wn), path in zip(got, want, ("graph", "plain launches")):
                print("%s, %s: %d launches, max |x0| %.4g" % (name, path, gn, float(g.abs().max())))
                assert bool(torch.isfinite(g).all()), (name, path)
                assert same(g, w), (name, path)
                assert gn == wn, (name, path, gn, wn)
    finally:
        eng.close()
