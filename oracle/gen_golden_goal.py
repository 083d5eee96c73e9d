"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/goal_frames.npz by running the UNMODIFIED reference's
recover_from_ric, get_target_location and recover_root_rot_heading_ang (data_loaders/humanml/scripts/motion_process.py)
on a synthetic chained motion:

    python -m oracle.gen_golden_goal

The fixture: B = 8 samples, one per joint configuration (the DIMP_FINAL options of get_allowed_joint_options, then
'heading' alone), goal joints ['pelvis'] + HML_EE_JOINT_NAMES as model_util gives them.  Each sample is a HumanML3D
feature sequence (263 features, those after the root-relative joints 0 once normalised) with non-zero yaw and root XZ
velocities, normalised with a synthetic mean / std, of three chunks of PRED frames, once after a CTX-frame prefix
("prefix": the returned motion of autoregressive_include_prefix) and once without ("noprefix").  Per case and chunk c (g_c = off + c * PRED):
  <case>_local_<c>  get_target_location(chunk c alone)                          [B, n_ext, 3]
  <case>_world_<c>  get_target_location(returned motion truncated after chunk c) [B, n_ext, 3]: the same joints at the
                    same frame, in W
plus <case>_motion [B, 263, N] (normalised), mean, std [263], is_heading [B], names (the joint lists, ';'-joined) and
the layout (ctx, pred, n_chunks).  tests/test_goal_chain_cpu.py checks that oracle/goal_oracle.py maps every world
entry onto the local one.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "goal_frames.npz")
D, CTX, PRED, N_CHUNKS = 263, 6, 12, 3


def _motion(rng, n):
    """[B, n, D] de-normalised features: a walk that keeps turning, with jittered root-relative joints"""
    B = 8
    x = rng.standard_normal((B, n, D)) * 0.05
    x[..., 0] = rng.uniform(-0.08, 0.08, (B, 1)) + 0.02 * rng.standard_normal((B, n))    # yaw velocity
    x[..., 1] = rng.uniform(-0.03, 0.03, (B, 1)) + 0.01 * rng.standard_normal((B, n))    # root x velocity
    x[..., 2] = rng.uniform(0.02, 0.06, (B, 1)) + 0.01 * rng.standard_normal((B, n))     # root z velocity
    x[..., 3] = 0.9 + 0.02 * rng.standard_normal((B, n))
    # hips and shoulders (joints 1, 2, 16, 17) well apart in x, so the heading is defined
    for j, dx in ((1, 0.1), (2, -0.1), (16, 0.18), (17, -0.18)):
        x[..., 4 + 3 * (j - 1)] += dx
    return x


def main():
    rh.load_reference()
    from data_loaders.humanml.scripts import motion_process as mp
    from data_loaders.humanml_utils import HML_EE_JOINT_NAMES
    rng = np.random.default_rng(7)
    names_all = ["pelvis"] + list(HML_EE_JOINT_NAMES)
    configs = mp.get_allowed_joint_options("DIMP_FINAL") + [["heading"]]
    names = [[j for j in c if j != "heading"] for c in configs]
    is_heading = torch.tensor(["heading" in c for c in configs])
    mean = rng.standard_normal(D).astype(np.float32) * 0.1
    std = rng.uniform(0.5, 1.5, D).astype(np.float32)
    mean[3] = 0.9
    m4, s4 = torch.from_numpy(mean)[None, :, None, None], torch.from_numpy(std)[None, :, None, None]
    out = dict(mean=mean, std=std, is_heading=is_heading.numpy(), names=np.array([";".join(n) for n in names]),
               ctx=np.int64(CTX), pred=np.int64(PRED), n_chunks=np.int64(N_CHUNKS))

    def target(motion):                                # motion [B, D, 1, n] normalised
        n = motion.shape[-1]
        lengths = torch.full((motion.shape[0],), n, dtype=torch.long)
        return mp.get_target_location(motion, m4, s4, lengths, 22, names_all, names, is_heading).numpy()

    for case, off in (("prefix", CTX), ("noprefix", 0)):
        n = off + N_CHUNKS * PRED
        raw = _motion(rng, n).astype(np.float32)
        norm = ((raw - mean) / std).astype(np.float32).transpose(0, 2, 1)       # [B, D, n]
        norm[:, 4 + 3 * 21:] = 0.0                     # features recover_from_ric does not read: kept small on disk
        motion = torch.from_numpy(norm)[:, :, None]
        out[case + "_motion"] = norm
        for c in range(N_CHUNKS):
            g = off + c * PRED
            out["%s_local_%d" % (case, c)] = target(motion[..., g:g + PRED])
            out["%s_world_%d" % (case, c)] = target(motion[..., :g + PRED])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
