"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/foot_contact.npz by running the UNMODIFIED reference's
extract_features (data_loaders/humanml/scripts/motion_process.py:43) on synthetic joint sequences:

    python -m oracle.gen_golden_foot

Skeletons: the reference's paramUtil (t2m_raw_offsets / t2m_kinematic_chain, kit_raw_offsets / kit_kinematic_chain);
face joints and feet as motion_process.py:462-464 (HumanML3D: fid_r [8, 11], fid_l [7, 10], face [2, 1, 17, 16]) and
:508-510 (KIT: fid_r [14, 15], fid_l [19, 20], face [11, 16, 5, 8]); threshold 0.002.  Each sequence is the skeleton's
forward kinematics under small smooth joint rotations, with a root that alternates between standing and walking, so the
feet are planted on some frames and slide on others.  Stored per dataset: <name>_features [T-1, D] fp32, <name>_contact
[T-1, 4] (the features' last four channels: feet_l, feet_r) and <name>_positions [T, J, 3] (the input positions), plus
`thres`.  tests/test_foot_guidance_cpu.py pins the derived contact mask, the channel-to-joint map and the (t, t+1) pair
convention to them.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "foot_contact.npz")
THRES = 0.002
T = 48
CASES = {"hml": dict(offsets="t2m_raw_offsets", chain="t2m_kinematic_chain", fid_r=[8, 11], fid_l=[7, 10],
                     face=[2, 1, 17, 16], seed=1),
         "kit": dict(offsets="kit_raw_offsets", chain="kit_kinematic_chain", fid_r=[14, 15], fid_l=[19, 20],
                     face=[11, 16, 5, 8], seed=2)}


def _sequence(skel_mod, quat_mod, offsets, chain, seed):
    """[T, J, 3] positions: forward kinematics of small smooth rotations, the root standing then walking"""
    rng = np.random.default_rng(seed)
    J = offsets.shape[0]
    skel = skel_mod.Skeleton(torch.from_numpy(offsets).float(), chain, "cpu")
    skel.set_offset(torch.from_numpy(offsets).float() * 0.3)
    t = np.arange(T)[:, None]
    angles = 0.25 * np.sin(2 * np.pi * (t / 24.0 + rng.random((1, J))))[..., None] * rng.standard_normal((1, J, 3))
    angles[:, 0] = 0.0
    quat = quat_mod.euler_to_quaternion(angles.reshape(-1, 3).astype(np.float64), "xyz").reshape(T, J, 4)
    speed = np.where((np.arange(T) // 12) % 2 == 0, 0.0, 0.06)
    root = np.stack([np.zeros(T), np.full(T, 0.9), np.cumsum(speed)], -1)
    pos = skel.forward_kinematics_np(quat, root)
    pos[..., 1] -= pos[..., 1].min()
    return pos


def main():
    rh.load_reference()
    if not hasattr(np, "float"):
        np.float = float          # extract_features' astype(np.float), removed from numpy 1.24
    from data_loaders.humanml.scripts import motion_process as mp
    from data_loaders.humanml.common import skeleton as skel_mod
    from data_loaders.humanml.common import quaternion as quat_mod
    from data_loaders.humanml.utils import paramUtil
    out = {"thres": np.float64(THRES)}
    for name, c in CASES.items():
        offsets, chain = getattr(paramUtil, c["offsets"]), getattr(paramUtil, c["chain"])
        pos = _sequence(skel_mod, quat_mod, offsets, chain, c["seed"])
        feats = mp.extract_features(pos.copy(), THRES, torch.from_numpy(offsets), chain, c["face"], c["fid_r"], c["fid_l"])
        out[name + "_features"] = feats.astype(np.float32)
        out[name + "_contact"] = feats[:, -4:].astype(np.float64)
        out[name + "_positions"] = pos.astype(np.float64)
        print(name, feats.shape, "contact share %.2f" % feats[:, -4:].mean())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
