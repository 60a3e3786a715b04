"""numpy restatement of pose_error_kernel (nope_b200/csrc/pose_error.cuh, DESIGN.md section 15), op by op in float64:
numpy's float64 multiply, add, subtract, divide and sqrt are the correctly rounded IEEE operations and are never
contracted, so the kernel's __dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn sequence is reproduced bit for bit when the
operations are applied in the same order.  Also the textbook formulas (np.linalg.norm of R @ x + t) the restatement is
checked against, and multi-tau VSD as render_oracle.vsd per tau."""
import numpy as np

from . import render_oracle


def _row(m, i, x, y, z):
    """((m_i0 x + m_i1 y) + m_i2 z) + m_i3; m [..., 3, 4] broadcast against the points"""
    return ((m[..., i, 0:1] * x + m[..., i, 1:2] * y) + m[..., i, 2:3] * z) + m[..., i, 3:4]


def compose(gt, sym):
    """gt [3, 4], sym [S, 3, 4] -> [S, 3, 4]: R_g R_s | R_g t_s + t_g, each entry ((g_i0 s_0j + g_i1 s_1j) + g_i2 s_2j)
    (+ tg_i for the translation column)"""
    g = np.asarray(gt, dtype=np.float64)
    s = np.asarray(sym, dtype=np.float64)
    out = (g[None, :, 0:1] * s[:, 0:1, :] + g[None, :, 1:2] * s[:, 1:2, :]) + g[None, :, 2:3] * s[:, 2:3, :]
    out[:, :, 3] = out[:, :, 3] + g[None, :, 3]
    return out


def pose_errors(points, sym, gt, est, K, chunk=64):
    """points [V, 3] float32, sym [S, 3, 4], gt [F, 3, 4], est [F, P, 3, 4], K [F, 4] -> (mssd, mspd) float64 [F, P]"""
    pts = np.asarray(points, dtype=np.float32).astype(np.float64)
    x, y, z = pts[None, :, 0], pts[None, :, 1], pts[None, :, 2]                # [1, V]
    sym, gt, est, K = (np.asarray(a, dtype=np.float64) for a in (sym, gt, est, K))
    F, P = est.shape[:2]
    mssd, mspd = np.full((F, P), np.inf), np.full((F, P), np.inf)
    for f in range(F):
        fx, fy, cx, cy = K[f]
        comp = compose(gt[f], sym)
        for p in range(P):
            e = est[f, p][None]
            ex, ey, ez = _row(e, 0, x, y, z), _row(e, 1, x, y, z), _row(e, 2, x, y, z)        # [1, V]
            bad_e = bool((~(ez > 0)).any())
            with np.errstate(divide="ignore", invalid="ignore"):
                eu = (fx * ex) / ez + cx
                ev = (fy * ey) / ez + cy
            for s0 in range(0, len(sym), chunk):
                c = comp[s0:s0 + chunk]
                gx, gy, gz = _row(c, 0, x, y, z), _row(c, 1, x, y, z), _row(c, 2, x, y, z)  # [s, V]
                dx, dy, dz = ex - gx, ey - gy, ez - gz
                me = ((dx * dx + dy * dy) + dz * dz).max(axis=1)
                with np.errstate(divide="ignore", invalid="ignore"):
                    du = eu - ((fx * gx) / gz + cx)
                    dv = ev - ((fy * gy) / gz + cy)
                    mp = np.fmax.reduce(du * du + dv * dv, axis=1)
                bad = (~(gz > 0)).any(axis=1) | bad_e
                mp = np.where(bad, np.inf, mp)
                mssd[f, p] = min(mssd[f, p], np.sqrt(me.min()))
                mspd[f, p] = min(mspd[f, p], np.sqrt(mp.min()))
    return mssd, mspd


def pose_errors_textbook(points, sym, gt, est, K):
    """the definitions with numpy's matrix products and norms (no control of rounding): (mssd, mspd) [F, P]"""
    pts = np.asarray(points, dtype=np.float32).astype(np.float64)
    sym, gt, est, K = (np.asarray(a, dtype=np.float64) for a in (sym, gt, est, K))
    F, P = est.shape[:2]
    mssd, mspd = np.zeros((F, P)), np.zeros((F, P))
    for f in range(F):
        fx, fy, cx, cy = K[f]
        for p in range(P):
            pe = pts @ est[f, p, :, :3].T + est[f, p, :, 3]
            best_s, best_p = np.inf, np.inf
            for s in sym:
                ps = pts @ s[:, :3].T + s[:, 3]
                pg = ps @ gt[f, :, :3].T + gt[f, :, 3]
                best_s = min(best_s, np.linalg.norm(pe - pg, axis=1).max())
                if (pe[:, 2] > 0).all() and (pg[:, 2] > 0).all():
                    ue = np.stack([fx * pe[:, 0] / pe[:, 2] + cx, fy * pe[:, 1] / pe[:, 2] + cy], axis=1)
                    ug = np.stack([fx * pg[:, 0] / pg[:, 2] + cx, fy * pg[:, 1] / pg[:, 2] + cy], axis=1)
                    best_p = min(best_p, np.linalg.norm(ue - ug, axis=1).max())
            mssd[f, p], mspd[f, p] = best_s, best_p
    return mssd, mspd


def vsd_taus(depth_test, depth_gt, depth_est, K, taus, delta=15, cost_type="step"):
    """float64 [P, T] for one frame: render_oracle.vsd at every tau"""
    return np.stack([render_oracle.vsd(depth_test, depth_gt, depth_est, K, delta, tau, cost_type) for tau in taus],
                    axis=1)
