"""TEST INFRASTRUCTURE ONLY -- the pose fits under occlusion of DESIGN.md section 24 restated in numpy, on top of the
unchanged oracles of the two fits.  An occluder mask O [H, W] (nonzero = something may be in front of the object)
leaves U = not O as the known pixels and the mask M' = M n U.

- The translation fit under O is translation_oracle.fit on a render whose O pixels read "no hit" (S' = S n U),
  against M'.
- The contour refinement under O is contour_refine_oracle.refine with phi and the box size of M', and a contour pixel
  counted and paired only when it and its four neighbours lie in U: `accumulate` restates that one rule and otherwise
  computes exactly contour_refine_oracle.accumulate.

`detection_occluders` restates nope_b200.crop.detection_occluders with a loop over the detections."""
import numpy as np

import contour_refine_oracle as cro
import translation_oracle as to

dro = cro.dro


def visible(mask, occ):
    """M' = M n U, bool"""
    return (np.asarray(mask) != 0) & (np.asarray(occ) == 0)


def hidden_render(render, occ):
    """the render callback with the O pixels read as "no hit" (depth 0)"""
    o = np.asarray(occ) != 0
    return lambda R, t: np.where(o, np.float32(0), np.asarray(render(R, t), dtype=np.float32))


# ------------------------------------------------------------------ translation
def fit_translation(render, R, t_init, mask, occ, K4, iters):
    """-> (t, iou, stats of S' at t) after `iters` updates of one hypothesis under O"""
    return to.fit(hidden_render(render, occ), R, t_init, visible(mask, occ), K4, iters)


def translation_stats(D, mask, occ):
    """stats(S', M') of one render D [H, W] (0 = not hit)"""
    o = np.asarray(occ) != 0
    return to.stats((np.asarray(D) > 0) & ~o, visible(mask, occ))


# ------------------------------------------------------------------ contour
def known4(occ):
    """bool [H, W]: the pixel and its four neighbours lie in U (the frame's border pixels are never contour pixels)"""
    u = np.asarray(occ) == 0
    out = u.copy()
    out[1:] &= u[:-1]
    out[:-1] &= u[1:]
    out[:, 1:] &= u[:, :-1]
    out[:, :-1] &= u[:, 1:]
    return out


def accumulate(D, phi, K4, t, tau, rho, occ):
    """contour_refine_oracle.accumulate with the contour restricted to known4(occ): -> (int64 [29] sums, n_contour)"""
    D = np.asarray(D, dtype=np.float32).astype(np.float64)
    phi = np.asarray(phi, dtype=np.float64)
    tau, rho = np.float64(tau), np.float64(rho)
    fx, fy = np.float64(K4[0]), np.float64(K4[1])
    cont = cro.contour(D) & known4(occ)
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
    k = cro.kappa(t[2], K4)
    n = [(au / z) * k, (av / z) * k, (-(((au * p[0] + av * p[1]) / z) / z)) * k]
    dp = [p[i] - np.float64(t[i]) for i in range(3)]
    J = [x / rho for x in dro._cross(dp, n)] + n
    et = e / tau
    sums = [dro.fixed(J[i] * J[j]).sum() for i, j in dro.UPPER]
    sums += [dro.fixed(J[i] * et).sum() for i in range(6)]
    sums += [dro.fixed(et * et).sum(), len(et)]
    return np.array(sums, dtype=np.int64), n_contour


def iou(D, mask, occ):
    """|S' n M'| / |S' u M'|; NaN for an M' without a contour (empty or full)"""
    o = np.asarray(occ) != 0
    return cro.iou(np.where(o, 0, np.asarray(D)), visible(mask, occ))


def refine_contour(render, R, t, mask, occ, K4, taus, rho):
    """-> (R, t, fit [4] = (n_in, n_contour, rms, iou), sums [29]) after len(taus) - 1 updates of one hypothesis
    under O, as contour_refine_oracle.refine"""
    R = np.array(R, dtype=np.float64)
    t = np.array(t, dtype=np.float64)
    mv = visible(mask, occ)
    phi, s = cro.sdf(mv), cro.box_size(mv)
    iters = len(taus) - 1
    for i in range(iters):
        tau = np.float64(taus[i]) * s
        sums, _ = accumulate(render(R, t), phi, K4, t, tau, rho, occ)
        R, t = cro.solve(sums, R, t, tau, K4, rho)
    D = render(R, t)
    tau = np.float64(taus[iters]) * s
    sums, nc = accumulate(D, phi, K4, t, tau, rho, occ)
    nin = float(int(sums[cro.NSUMS - 1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        rms = tau * np.sqrt(np.float64(dro.unfix(sums[cro.NSUMS - 2])) / np.float64(nin))
    return R, t, np.array([nin, float(nc), rms, iou(D, mask, occ)]), sums


# ------------------------------------------------------------------ occluders from a frame's detections
def detection_occluders(masks, frame_idx):
    """uint8 [B, H, W]: the union of the other detections' masks of the same frame, minus the detection's own"""
    m = np.asarray(masks) != 0
    fi = np.asarray(frame_idx)
    out = np.zeros(m.shape, dtype=np.uint8)
    for b in range(len(m)):
        others = [j for j in range(len(m)) if j != b and fi[j] == fi[b]]
        if others:
            out[b] = m[others].any(0) & ~m[b]
    return out
