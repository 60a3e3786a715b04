"""TEST INFRASTRUCTURE ONLY -- the contour refinement of nope_b200/csrc/contour_refine.cuh (DESIGN.md section 20)
restated in numpy float64, in the kernel's operation order.  numpy's elementwise float64 multiply, add, divide and sqrt
are the IEEE operations and are never contracted, the fixed-point products are summed as int64, and the solve is
depth_refine_oracle.solve at the metric tolerance, so the kernel matches this bit for bit.

The distance transform here is the definition itself: the column distances by two running scans, then for every
pixel the minimum over the columns of its row by widening offsets, stopped once the offset alone exceeds the largest
minimum found.  The renderer is a callback render(R [3, 3] float64, t [3] float64) -> depth [H, W] (0 where nothing is
hit), as in depth_refine_oracle."""
import numpy as np

import depth_refine_oracle as dro
import translation_oracle as to

NSUMS = dro.NSUMS
_INF = np.int64(1) << 40


def _column_distance(feature):
    """int64 [H, W]: the row distance to the nearest True pixel of the same column, _INF when the column has none"""
    H, W = feature.shape
    rows = np.arange(H, dtype=np.int64)[:, None]
    above = np.maximum.accumulate(np.where(feature, rows, -_INF), axis=0)
    below = np.minimum.accumulate(np.where(feature, rows, _INF)[::-1], axis=0)[::-1]
    return np.where(feature.any(0)[None], np.minimum(rows - above, below - rows), _INF)


def _row_minimum(gcol):
    """int64 [H, W]: min over columns c' of (c - c')^2 + gcol(r, c')^2 (_INF where every gcol of the row is _INF)"""
    H, W = gcol.shape
    g2 = np.where(gcol >= _INF, _INF, gcol * gcol)
    d2 = g2.copy()
    for k in range(1, W):
        if k * k >= d2.max():
            break
        d2[:, k:] = np.minimum(d2[:, k:], g2[:, :-k] + k * k)
        d2[:, :-k] = np.minimum(d2[:, :-k], g2[:, k:] + k * k)
    return np.minimum(d2, _INF)


def sq_distances(mask):
    """(d2_out, d2_in) int64 [H, W] of one mask: the squared distance to the nearest object / background pixel of the
    frame, -1 where the frame has none"""
    m = np.asarray(mask) != 0
    out = []
    for feature in (m, ~m):
        d2 = _row_minimum(_column_distance(feature)) if feature.any() else np.full(m.shape, _INF)
        out.append(np.where(d2 >= _INF, -1, d2))
    return out[0], out[1]


def sdf(mask):
    """phi float64 [H, W]: sqrt(d2_out) - 1/2 off the object, 1/2 - sqrt(d2_in) on it; NaN for an empty or full mask"""
    m = np.asarray(mask) != 0
    if not m.any() or m.all():
        return np.full(m.shape, np.nan)
    d2_out, d2_in = sq_distances(m)
    return np.where(m, 0.5 - np.sqrt(d2_in.astype(np.float64)), np.sqrt(d2_out.astype(np.float64)) - 0.5)


def box_size(mask):
    """s = sqrt(w h) of the mask's bounding box; NaN for a mask without a contour (empty or full)"""
    m = np.asarray(mask) != 0
    if not m.any() or m.all():
        return np.float64(np.nan)
    n, _, r0, r1, c0, c1 = to.stats(m)
    return np.sqrt(np.float64(c1 - c0 + 1) * np.float64(r1 - r0 + 1))


def kappa(t2, K4):
    """t_2 / sqrt(fx fy)"""
    return np.float64(t2) / np.sqrt(np.float64(K4[0]) * np.float64(K4[1]))


def contour(D):
    """bool [H, W]: the interior pixels of the render D (0 = not hit) that are hit and have a 4-neighbour not hit"""
    D = np.asarray(D, dtype=np.float32)
    hit = D > 0
    H, W = D.shape
    out = np.zeros((H, W), dtype=bool)
    c_, r_ = slice(1, W - 1), slice(1, H - 1)
    out[r_, c_] = hit[r_, c_] & ~(hit[r_, 2:] & hit[r_, :-2] & hit[2:, c_] & hit[:-2, c_])
    return out


def visible(mask, occ):
    """M' = M n U, bool: the mask's pixels outside the occluder mask occ (nonzero = something may be in front)"""
    return (np.asarray(mask) != 0) & (np.asarray(occ) == 0)


def known4(occ):
    """bool [H, W]: the pixel and its four neighbours lie in U = not occ (the frame's border pixels are never contour
    pixels)"""
    u = np.asarray(occ) == 0
    out = u.copy()
    out[1:] &= u[:-1]
    out[:-1] &= u[1:]
    out[:, 1:] &= u[:, :-1]
    out[:, :-1] &= u[:, 1:]
    return out


def accumulate(D, phi, K4, t, tau, rho, occ=None):
    """-> (int64 [29] sums, n_contour) of one render D [H, W] against the mask's phi [H, W] at the pixel tolerance tau:
    the 21 entries of the upper triangle of J J^T row by row, the 6 of J e, e^2 and the pair count.  With an occluder
    mask occ, a contour pixel is counted and paired only when it and its four neighbours lie in U (known4)."""
    D = np.asarray(D, dtype=np.float32).astype(np.float64)
    phi = np.asarray(phi, dtype=np.float64)
    tau, rho = np.float64(tau), np.float64(rho)
    fx, fy = np.float64(K4[0]), np.float64(K4[1])
    cont = contour(D) if occ is None else contour(D) & known4(occ)
    n_contour = int(cont.sum())
    r, c = np.nonzero(cont)
    e = phi[r, c] + 0.5
    with np.errstate(invalid="ignore"):
        keep = np.abs(e) <= tau
    r, c, e = r[keep], c[keep], e[keep]
    gu = (phi[r, c + 1] - phi[r, c - 1]) * 0.5
    gv = (phi[r + 1, c] - phi[r - 1, c]) * 0.5
    keep = ~((gu == 0) & (gv == 0))
    r, c, e, gu, gv = r[keep], c[keep], e[keep], gu[keep], gv[keep]
    p = dro._point(r, c, D[r, c], K4)
    z = p[2]
    au, av = gu * fx, gv * fy
    k = kappa(t[2], K4)
    n = [(au / z) * k, (av / z) * k, (-(((au * p[0] + av * p[1]) / z) / z)) * k]
    dp = [p[i] - np.float64(t[i]) for i in range(3)]
    J = [x / rho for x in dro._cross(dp, n)] + n
    et = e / tau
    sums = [dro.fixed(J[i] * J[j]).sum() for i, j in dro.UPPER]
    sums += [dro.fixed(J[i] * et).sum() for i in range(6)]
    sums += [dro.fixed(et * et).sum(), len(et)]
    return np.array(sums, dtype=np.int64), n_contour


def solve(sums, R, t, tau, K4, rho):
    """one update at the pixel tolerance tau: depth_refine_oracle.solve at tau_m = tau kappa; t_2 <= 0 keeps the pose"""
    if not np.float64(t[2]) > 0:
        return np.array(R, dtype=np.float64), np.array(t, dtype=np.float64)
    return dro.solve(sums, R, t, np.float64(tau) * kappa(t[2], K4), rho)


def iou(D, mask, occ=None):
    """|S n M| / |S u M| of the render's silhouette and the mask; NaN for a mask without a contour.  With an occluder
    mask occ: |S' n M'| / |S' u M'| of both restricted to U."""
    m = np.asarray(mask) != 0
    if occ is not None:
        D, m = np.where(np.asarray(occ) != 0, 0, np.asarray(D)), visible(mask, occ)
    if not m.any() or m.all():
        return np.nan
    return to.iou(to.stats(np.asarray(D) > 0, m), to.stats(m))


def refine(render, R, t, mask, K4, taus, rho, phi=None, occ=None):
    """-> (R, t, fit [4] = (n_in, n_contour, rms, iou), sums [29]) after len(taus) - 1 updates of one hypothesis,
    iteration i pairing at taus[i] times the mask's box size.  Under an occluder mask occ, phi and the box size are
    those of M' = visible(mask, occ), and accumulate and iou leave the occluded pixels out."""
    R = np.array(R, dtype=np.float64)
    t = np.array(t, dtype=np.float64)
    mv = mask if occ is None else visible(mask, occ)
    phi = sdf(mv) if phi is None else phi
    s = box_size(mv)
    iters = len(taus) - 1
    for i in range(iters):
        tau = np.float64(taus[i]) * s
        sums, _ = accumulate(render(R, t), phi, K4, t, tau, rho, occ)
        R, t = solve(sums, R, t, tau, K4, rho)
    D = render(R, t)
    tau = np.float64(taus[iters]) * s
    sums, nc = accumulate(D, phi, K4, t, tau, rho, occ)
    nin = float(int(sums[NSUMS - 1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        rms = tau * np.sqrt(np.float64(dro.unfix(sums[NSUMS - 2])) / np.float64(nin))
    return R, t, np.array([nin, float(nc), rms, iou(D, mask, occ)]), sums
