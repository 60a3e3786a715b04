"""Float64 oracle of the distinct top-k (DESIGN.md section 21; csrc/distinct.cuh).  Every step is one numpy
elementwise operation (correctly rounded, never contracted) in the kernel's order, so the kernel must match it bit for
bit.  No import from the product."""
import math

import numpy as np


def closeness(Ri, Rj, D, axis):
    """c(i, j) for one selected rotation Ri [3, 3] and candidates Rj [..., 3, 3] under the group (D [n, 3, 3] with
    D[0] the identity, axis [3], zeros for none) -> float64 [..., n], one value per discrete rotation d (c is their
    maximum).  P = Rj^T Ri, M_d = D_d P; tr M_d, or with an axis a^T M_d a + sqrt((tr M_d - a^T M_d a)^2 + s^2)."""
    Ri, Rj, D = np.asarray(Ri, np.float64), np.asarray(Rj, np.float64), np.asarray(D, np.float64)
    P = np.empty(Rj.shape[:-2] + (3, 3))
    for a in range(3):
        for b in range(3):
            P[..., a, b] = Rj[..., 0, a] * Ri[0, b] + Rj[..., 1, a] * Ri[1, b] + Rj[..., 2, a] * Ri[2, b]
    out = np.empty(Rj.shape[:-2] + (len(D),))
    has_axis = bool(np.any(np.asarray(axis) != 0))
    ax = np.asarray(axis, np.float64)
    for d in range(len(D)):
        M = np.empty_like(P)
        for a in range(3):
            for b in range(3):
                M[..., a, b] = D[d, a, 0] * P[..., 0, b] + D[d, a, 1] * P[..., 1, b] + D[d, a, 2] * P[..., 2, b]
        t = M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2]
        if not has_axis:
            out[..., d] = t
            continue
        v = [M[..., a, 0] * ax[0] + M[..., a, 1] * ax[1] + M[..., a, 2] * ax[2] for a in range(3)]
        u = ax[0] * v[0] + ax[1] * v[1] + ax[2] * v[2]
        s = ax[0] * (M[..., 2, 1] - M[..., 1, 2]) + ax[1] * (M[..., 0, 2] - M[..., 2, 0]) + \
            ax[2] * (M[..., 1, 0] - M[..., 0, 1])
        w = t - u
        out[..., d] = u + np.sqrt(w * w + s * s)
    return out


def threshold(min_angle_deg):
    """c_thr = 1 + 2 cos(theta), with Python's float64 cos as the host computes it"""
    return 1.0 + 2.0 * math.cos(math.radians(float(min_angle_deg)))


def distinct_row(sim, rot, k, c_thr, D, axis):
    """One row: sim [N] float32, rot [N, 3, 3] -> (score float32 [k], idx int64 [k]).  Greedy in the order of a stable
    sort of -score; -inf and NaN never taken; an entry is dropped once some c_d(pick, entry) >= c_thr."""
    sim = np.asarray(sim, np.float32)
    alive = sim > -np.inf                                     # False for -inf and NaN
    order = np.argsort(-sim.astype(np.float64), kind="stable")
    score, idx = np.full(k, -np.inf, np.float32), np.full(k, -1, np.int64)
    pos = 0
    for t in range(k):
        while pos < len(order) and not alive[order[pos]]:
            pos += 1
        if pos == len(order):
            break
        i = int(order[pos])
        score[t], idx[t] = sim[i], i
        alive[i] = False
        rest = np.nonzero(alive)[0]
        if len(rest):
            alive[rest[(closeness(rot[i], rot[rest], D, axis) >= c_thr).any(axis=-1)]] = False
    return score, idx


def distinct_topk(sim, rot, k, c_thr, groups, group, Q=None):
    """sim [R, N], rot [G_r, N, 3, 3] (row r uses rot[r // Q], or rot[0] when G_r = 1), groups [(D, axis)], group [R]
    -> (score [R, k], idx [R, k])"""
    sim = np.asarray(sim, np.float32)
    R = sim.shape[0]
    G_r = rot.shape[0]
    Q = R // G_r if Q is None else Q
    out = [distinct_row(sim[r], rot[0 if G_r == 1 else r // Q], k, c_thr, *groups[group[r]]) for r in range(R)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])
