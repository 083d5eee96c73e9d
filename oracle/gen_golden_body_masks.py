"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/hml_body_masks.npz from the UNMODIFIED reference's HumanML3D
body-part masks (data_loaders/humanml_utils.py: HML_LOWER_BODY_MASK, HML_UPPER_BODY_MASK, bool [263]):

    python -m oracle.gen_golden_body_masks

tests/test_multi_prompt_cpu.py pins b200mdm.body_part_mask to them.
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "hml_body_masks.npz")


def main():
    path = os.path.join(rh.REFERENCE_ROOT, "data_loaders", "humanml_utils.py")
    spec = importlib.util.spec_from_file_location("ref_humanml_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    np.savez_compressed(OUT, lower=np.asarray(mod.HML_LOWER_BODY_MASK, dtype=bool),
                        upper=np.asarray(mod.HML_UPPER_BODY_MASK, dtype=bool))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
