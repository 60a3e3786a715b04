"""numpy float64 restatement of track_seed_kernel (nope_b200/csrc/track.cuh), op by op: every product, sum, division
and sqrt rounded on its own, as numpy's elementwise float64 operations are."""
import numpy as np


def residuals(Rc, T):
    """M [H, N, 3, 3] = Rc T^T, each entry ((Rc_i0 T_j0 + Rc_i1 T_j1) + Rc_i2 T_j2)"""
    Rc = np.asarray(Rc, dtype=np.float64)[:, None]
    T = np.asarray(T, dtype=np.float64)[None]
    M = np.empty(np.broadcast_shapes(Rc.shape, T.shape))
    with np.errstate(invalid="ignore"):
        for i in range(3):
            for j in range(3):
                M[..., i, j] = (Rc[..., i, 0] * T[..., j, 0] + Rc[..., i, 1] * T[..., j, 1]) + \
                    Rc[..., i, 2] * T[..., j, 2]
    return M


def scores(M):
    """-> (a, b, r, score) of residuals M [..., 3, 3]"""
    a = M[..., 0, 0] + M[..., 1, 1]
    b = M[..., 1, 0] - M[..., 0, 1]
    with np.errstate(invalid="ignore"):
        r = np.sqrt(a * a + b * b)
    return a, b, r, r + M[..., 2, 2]


def track_seeds(Rc, T):
    """Rc [H, 3, 3], T [N, 3, 3] float64 -> (D [H, 3, 3] float32, seed [H] int32, cossin [H, 2] float32)"""
    Rc = np.asarray(Rc, dtype=np.float64).reshape(-1, 3, 3)
    T = np.asarray(T, dtype=np.float64).reshape(-1, 3, 3)
    H = Rc.shape[0]
    M = residuals(Rc, T)
    _, _, _, s = scores(M)
    D = np.tile(np.eye(3, dtype=np.float32), (H, 1, 1))
    seed = np.zeros(H, dtype=np.int32)
    cs = np.tile(np.array([1.0, 0.0], dtype=np.float32), (H, 1))
    for h in range(H):
        valid = ~np.isnan(s[h])
        if not np.isfinite(Rc[h]).all() or not valid.any():
            continue
        best = np.max(s[h][valid])
        n = int(np.flatnonzero(valid & (s[h] == best))[0])         # ties -> the lowest n
        m = M[h, n]
        a, b, r, _ = scores(m)
        c, sn = (1.0, 0.0) if r == 0.0 else (a / r, b / r)
        d = np.empty((3, 3))
        for j in range(3):
            d[0, j] = c * m[0, j] + sn * m[1, j]
            d[1, j] = c * m[1, j] - sn * m[0, j]
            d[2, j] = m[2, j]
        D[h], seed[h], cs[h] = d.astype(np.float32), n, np.array([c, sn]).astype(np.float32)
    return D, seed, cs


def compose(D, seed, cossin, T):
    """Rz(rho) D T[seed] in float64 of the float32 outputs"""
    c, s = np.asarray(cossin, dtype=np.float64)[..., 0], np.asarray(cossin, dtype=np.float64)[..., 1]
    Rz = np.zeros(c.shape + (3, 3))
    Rz[..., 0, 0], Rz[..., 0, 1], Rz[..., 1, 0], Rz[..., 1, 1], Rz[..., 2, 2] = c, -s, s, c, 1.0
    return Rz @ np.asarray(D, dtype=np.float64) @ np.asarray(T, dtype=np.float64)[seed]


def random_rotations(n, rng):
    q = rng.standard_normal((n, 4))
    w, x, y, z = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3)


def rz(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), -np.sin(t), 0.0], [np.sin(t), np.cos(t), 0.0], [0.0, 0.0, 1.0]])
