"""TEST INFRASTRUCTURE ONLY -- the depth refinement of nope_b200/csrc/depth_refine.cuh (DESIGN.md section 19) restated
in numpy float64, in the kernel's operation order.  numpy's elementwise float64 multiply, add, divide and sqrt are the
IEEE operations and are never contracted, the fixed-point products are summed as int64, and the solve runs on Python
floats one operation at a time, so the kernel matches this bit for bit.

The renderer is a callback render(R [3, 3] float64, t [3] float64) -> depth [H, W] (0 where nothing is hit);
`translation_oracle.cpu_renderer` wraps oracle/render_oracle.render, and GPU tests pass nope_b200.vsd.render_depth
images."""
import math

import numpy as np

NSUMS = 29
SCALE = 2.0 ** 32            # one fixed-point unit is 2^-32
CLAMP = 16.0                 # |product| <= 16 before the conversion
DAMPING = 1e-2               # mu = DAMPING max diag(A)
UPPER = [(a, b) for a in range(6) for b in range(a, 6)]


def fixed(x):
    """per-pixel products -> int64 fixed point: clamped to [-16, 16], times 2^32, rounded half to even"""
    return np.rint(np.clip(np.asarray(x, dtype=np.float64), -CLAMP, CLAMP) * SCALE).astype(np.int64)


def unfix(s):
    return float(int(s)) * (1.0 / SCALE)


def _point(r, c, z, K4):
    """X(r, c, z) = ((c + 1/2 - cx) z / fx, (r + 1/2 - cy) z / fy, z)"""
    fx, fy, cx, cy = (np.float64(v) for v in K4)
    c = np.asarray(c, dtype=np.float64)
    r = np.asarray(r, dtype=np.float64)
    return [((c + 0.5) - cx) * z / fx, ((r + 0.5) - cy) * z / fy, z]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def valid_count(S, mask=None):
    """n_valid: the pixels with a sensor reading inside the mask"""
    S = np.asarray(S, dtype=np.float64)
    ok = S > 0
    if mask is not None:
        ok &= np.asarray(mask) != 0
    return int(ok.sum())


def accumulate(D, S, mask, K4, t, tau, rho):
    """int64 [29] sums of one render D [H, W] (0 = not hit) against the sensor depth S [H, W]: the 21 entries of the
    upper triangle of J J^T row by row, the 6 of J e, e^2 and the pair count"""
    D = np.asarray(D, dtype=np.float32).astype(np.float64)
    S = np.asarray(S, dtype=np.float64)
    H, W = D.shape
    tau, rho = np.float64(tau), np.float64(rho)
    ok = np.zeros((H, W), dtype=bool)
    c_ = slice(1, W - 1)
    r_ = slice(1, H - 1)
    d, s = D[r_, c_], S[r_, c_]
    with np.errstate(invalid="ignore"):
        ok[r_, c_] = (d > 0) & (D[r_, 2:] > 0) & (D[r_, :-2] > 0) & (D[2:, c_] > 0) & (D[:-2, c_] > 0) & (s > 0) \
            & (np.abs(s - d) <= tau)
    if mask is not None:
        ok &= np.asarray(mask) != 0
    r, c = np.nonzero(ok)
    d, s = D[r, c], S[r, c]
    p = _point(r, c, d, K4)
    q = _point(r, c, s, K4)
    a, b = _point(r, c + 1, D[r, c + 1], K4), _point(r, c - 1, D[r, c - 1], K4)
    eu = [a[k] - b[k] for k in range(3)]
    a, b = _point(r + 1, c, D[r + 1, c], K4), _point(r - 1, c, D[r - 1, c], K4)
    ev = [a[k] - b[k] for k in range(3)]
    nr = _cross(eu, ev)
    len2 = _dot(nr, nr)
    keep = len2 != 0
    p, q, nr, len2 = [x[keep] for x in p], [x[keep] for x in q], [x[keep] for x in nr], len2[keep]
    ln = np.sqrt(len2)
    n = [nr[k] / ln for k in range(3)]
    flip = _dot(n, p) > 0
    n = [np.where(flip, -n[k], n[k]) for k in range(3)]
    dp = [p[k] - np.float64(t[k]) for k in range(3)]
    J = [x / rho for x in _cross(dp, n)] + n
    e = _dot(n, [p[k] - q[k] for k in range(3)]) / tau
    sums = [fixed(J[i] * J[j]).sum() for i, j in UPPER]
    sums += [fixed(J[i] * e).sum() for i in range(6)]
    sums += [fixed(e * e).sum(), len(e)]
    return np.array(sums, dtype=np.int64)


def solve(sums, R, t, tau, rho):
    """one update of (R [3, 3], t [3]) from the sums; n_in < 6 or a non-positive pivot -> unchanged"""
    R = np.array(R, dtype=np.float64)
    t = np.array(t, dtype=np.float64)
    if int(sums[NSUMS - 1]) < 6:
        return R, t
    M = [[0.0] * 6 for _ in range(6)]
    for q, (a, b) in enumerate(UPPER):
        M[a][b] = M[b][a] = unfix(sums[q])
    g = [unfix(sums[21 + a]) for a in range(6)]
    dmax = max(M[a][a] for a in range(6))
    mu = DAMPING * dmax
    for a in range(6):
        M[a][a] = M[a][a] + mu
    L = [[0.0] * 6 for _ in range(6)]
    for j in range(6):
        x = M[j][j]
        for k in range(j):
            x = x - L[j][k] * L[j][k]
        if not x > 0.0:
            return R, t
        L[j][j] = math.sqrt(x)
        for r in range(j + 1, 6):
            x = M[r][j]
            for k in range(j):
                x = x - L[r][k] * L[j][k]
            L[r][j] = x / L[j][j]
    y = [0.0] * 6
    for r in range(6):
        x = -g[r]
        for k in range(r):
            x = x - L[r][k] * y[k]
        y[r] = x / L[r][r]
    dl = [0.0] * 6
    for r in range(5, -1, -1):
        x = y[r]
        for k in range(r + 1, 6):
            x = x - L[k][r] * dl[k]
        dl[r] = x / L[r][r]
    tau, rho = float(tau), float(rho)
    h = [dl[k] * tau / rho * 0.5 for k in range(3)]
    sn = math.sqrt(1.0 + ((h[0] * h[0] + h[1] * h[1]) + h[2] * h[2]))
    qw, qx, qy, qz = 1.0 / sn, h[0] / sn, h[1] / sn, h[2] / sn
    xx, yy, zz, xy, xz, yz = qx * qx, qy * qy, qz * qz, qx * qy, qx * qz, qy * qz
    wx, wy, wz = qw * qx, qw * qy, qw * qz
    Rd = [[1.0 - 2.0 * (yy + zz), 2.0 * (xy - wz), 2.0 * (xz + wy)],
          [2.0 * (xy + wz), 1.0 - 2.0 * (xx + zz), 2.0 * (yz - wx)],
          [2.0 * (xz - wy), 2.0 * (yz + wx), 1.0 - 2.0 * (xx + yy)]]
    Rn = np.array([[(Rd[r][0] * float(R[0, c]) + Rd[r][1] * float(R[1, c])) + Rd[r][2] * float(R[2, c])
                    for c in range(3)] for r in range(3)])
    tn = np.array([float(t[k]) + dl[3 + k] * tau for k in range(3)])
    return Rn, tn


def fit_stats(sums, n_valid, tau):
    """(n_in, n_valid, rms, score) of the sums of the last render"""
    nin = float(int(sums[NSUMS - 1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        rms = np.float64(tau) * np.sqrt(np.float64(unfix(sums[NSUMS - 2])) / np.float64(nin))
        score = np.float64(nin) / np.float64(n_valid)
    return np.array([nin, float(n_valid), rms, score])


def refine(render, R, t, S, mask, K4, taus, rho):
    """-> (R, t, fit [4], sums [29]) after len(taus) - 1 updates of one hypothesis, iteration i pairing at taus[i]"""
    R = np.array(R, dtype=np.float64)
    t = np.array(t, dtype=np.float64)
    iters = len(taus) - 1
    for i in range(iters):
        R, t = solve(accumulate(render(R, t), S, mask, K4, t, taus[i], rho), R, t, taus[i], rho)
    sums = accumulate(render(R, t), S, mask, K4, t, taus[iters], rho)
    return R, t, fit_stats(sums, valid_count(S, mask), taus[iters]), sums


def radius(vertices):
    """rho: the largest vertex norm, float64 of the float32 vertices"""
    v = np.asarray(vertices, dtype=np.float32).astype(np.float64)
    return float(np.sqrt((v * v).sum(1)).max())
