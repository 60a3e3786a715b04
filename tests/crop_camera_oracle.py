"""The crop camera (DESIGN.md section 23) restated op by op in float64, as crop_camera_kernel and crop_rotate_kernel
(nope_b200/csrc/crop.cuh) compute it: every product, sum, quotient and square root rounded on its own (Python floats
and math.sqrt are IEEE float64, correctly rounded, and never contracted), norms sqrt((a a + b b) + c c), divisions per
component, matrix entries (p0 + p1) + p2.  The kernels must equal this bit for bit."""
import math

import numpy as np


def _norm(a, b, c):
    return math.sqrt((a * a + b * b) + c * c)


def _vectors(pose, keep_inplane):
    """crop_frame's `upper` and `right` (nope_b200.crop._corners) of one pose [4, 4]"""
    ox, oy, oz = float(pose[0, 3]), float(pose[1, 3]), float(pose[2, 3])
    if keep_inplane:
        upper = (0.0, -oz, oy)
        right = (oy * oy + oz * oz, -(ox * oy), -(ox * oz))
    else:
        a = (0.0 - ox, 0.0 - oy, 6.0 - oz)
        up = [((float(pose[i, 0]) * a[0] + float(pose[i, 1]) * a[1]) + float(pose[i, 2]) * a[2]) + float(pose[i, 3])
              for i in range(3)]
        right = (oy * up[2] - oz * up[1], oz * up[0] - ox * up[2], ox * up[1] - oy * up[0])
        rx, ry, rz = right
        upper = (ry * oz - rz * oy, rz * ox - rx * oz, rx * oy - ry * ox)
    return (ox, oy, oz), upper, right


def crop_camera(pose, keep_inplane=True):
    """R_v float64 [F, 3, 3] of poses [F, 4, 4] (or [4, 4] -> [3, 3])"""
    P = np.asarray(pose, dtype=np.float64)
    one = P.ndim == 2
    P = P.reshape(-1, 4, 4)
    out = np.empty((len(P), 3, 3))
    for f, p in enumerate(P):
        o, upper, right = _vectors(p, keep_inplane)
        nu, nr, no = _norm(*upper), _norm(*right), _norm(*o)
        if nu == 0.0 and nr == 0.0:
            out[f] = np.eye(3)
            continue
        out[f, 0] = [r / nr for r in right]
        out[f, 1] = [-(u / nu) for u in upper]
        out[f, 2] = [c / no for c in o]
    return out[0] if one else out


def crop_rotate(Rv, R, to_camera):
    """Rv [F, 3, 3], R [F, P, 3, 3] -> Rv^T R (to_camera) or Rv R, float64 [F, P, 3, 3]"""
    Rv = np.asarray(Rv, dtype=np.float64)
    R = np.asarray(R, dtype=np.float64)
    out = np.empty(R.shape)
    for f in range(R.shape[0]):
        A = Rv[f].T if to_camera else Rv[f]
        for p in range(R.shape[1]):
            r = R[f, p]
            for i in range(3):
                for j in range(3):
                    out[f, p, i, j] = (float(A[i, 0]) * float(r[0, j]) + float(A[i, 1]) * float(r[1, j])) + \
                        float(A[i, 2]) * float(r[2, j])
    return out


def intrinsics(pose, virtual_bbox_size, image_size):
    """K_v [3, 3] of one pose: f_v = S |o| / s, principal point (S/2, S/2)"""
    o = np.asarray(pose, dtype=np.float64)[:3, 3]
    f = image_size * _norm(*map(float, o)) / virtual_bbox_size
    return np.array([[f, 0.0, image_size / 2], [0.0, f, image_size / 2], [0.0, 0.0, 1.0]])


def seeded_poses(seed, F, keep_inplane, K=None, W=720, H=540):
    """F poses [F, 4, 4]: object centres 400 ... 1200 mm deep, projecting anywhere in a W x H frame of intrinsics K
    (Primesense by default), random rotations (the keep_inplane=False mode reads them)"""
    from scipy.spatial.transform import Rotation
    K = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]]) if K is None else K
    rng = np.random.default_rng(seed)
    out = np.tile(np.eye(4), (F, 1, 1))
    z = rng.uniform(400.0, 1200.0, F)
    u, v = rng.uniform(0, W, F), rng.uniform(0, H, F)
    out[:, 0, 3] = (u - K[0, 2]) * z / K[0, 0]
    out[:, 1, 3] = (v - K[1, 2]) * z / K[1, 1]
    out[:, 2, 3] = z
    if not keep_inplane:
        out[:, :3, :3] = Rotation.random(F, random_state=rng).as_matrix()
    return out
