"""TEST INFRASTRUCTURE ONLY -- write tests/golden/inplane.npz from the UNMODIFIED reference's own in-plane helpers
(`adding_inplane_to_pose` / `compute_inplane`, src/poses/utils.py:295-315) applied to its level-2 template poses
(src/poses/predefined_poses/obj_poses_level2.npy) at seeded grid angles alpha = a * 360 / A.  Per sample: the template
rotation T, A, the angle index a, alpha in degrees, query_R = adding_inplane_to_pose(T, inplane=-alpha) and
inplane = compute_inplane(query_R, T).  Writes this one fixture and nothing else.

Run in the build container (CPU):   python -m oracle.make_inplane
"""
import json
import os
import sys

import numpy as np

from . import inputs
from .ref_import import REFERENCE_ROOT, _install_stubs


def write_inplane(out_dir=inputs.GOLDEN_DIR, n=24, seed=0):
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    from src.poses.utils import adding_inplane_to_pose, compute_inplane
    poses = np.load(os.path.join(REFERENCE_ROOT, "src/poses/predefined_poses/obj_poses_level2.npy"))
    rng = np.random.default_rng(seed)
    level2_idx = rng.choice(len(poses), size=n, replace=False)
    A = rng.choice([4, 7, 12, 36, 360], size=n)
    a = np.array([rng.integers(0, A_) for A_ in A])
    alpha = a * 360.0 / A
    T = poses[level2_idx, :3, :3].astype(np.float64)
    query_R = np.stack([adding_inplane_to_pose(T[i], -alpha[i]) for i in range(n)])
    inplane = np.array([compute_inplane(query_R[i], T[i]) for i in range(n)])
    np.savez_compressed(os.path.join(out_dir, "inplane.npz"), level2_idx=level2_idx.astype(np.int64),
                        template_R=T, A=A.astype(np.int64), angle_idx=a.astype(np.int64), alpha_deg=alpha,
                        query_R=query_R, inplane=inplane)
    return {"samples": n, "A": sorted(set(A.tolist()))}


def main():
    print(json.dumps(write_inplane(), indent=1))


if __name__ == "__main__":
    sys.exit(main())
