"""TEST INFRASTRUCTURE ONLY -- write tests/golden/pose_nesting.npz from the UNMODIFIED reference's shipped
nesting of its level-0 pose grids in the level-2 grid (src/poses/predefined_poses/idx_{all,upper}_level0_in_level2.npy,
read by src/dataloader/shapeNet.py:252-263 for its fast evaluation), as data.  Both arrays index the level-2 'all'
grid: entry i is the level-2 pose nearest to level-0 pose i.  Writes this one fixture and nothing else.

Run in the build container (CPU):   python -m oracle.make_nesting
"""
import json
import os
import sys

import numpy as np

from . import inputs
from .ref_import import REFERENCE_ROOT


def write_pose_nesting(out_dir=inputs.GOLDEN_DIR):
    pp = os.path.join(REFERENCE_ROOT, "src/poses/predefined_poses")
    out = {f"idx_{d}_level0_in_level2": np.load(os.path.join(pp, f"idx_{d}_level0_in_level2.npy")).astype(np.int64)
           for d in ("all", "upper")}
    np.savez_compressed(os.path.join(out_dir, "pose_nesting.npz"), **out)
    return {k: v.shape[0] for k, v in out.items()}


def main():
    print(json.dumps(write_pose_nesting(), indent=1))


if __name__ == "__main__":
    sys.exit(main())
