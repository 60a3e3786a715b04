"""TEST INFRASTRUCTURE ONLY -- the translation fit of nope_b200/csrc/translation.cuh (DESIGN.md section 18) restated in
numpy float64, in the kernel's operation order.  numpy's float64 multiply, add, divide and sqrt are the IEEE
operations and are never contracted, so the kernel matches this bit for bit.

The renderer is a callback render(R [3, 3] float64, t [3] float64) -> depth [H, W]; `cpu_renderer` wraps
oracle/render_oracle.render, and GPU tests pass nope_b200.vsd.render_depth images."""
import numpy as np

from oracle import render_oracle as ro


def stats(image, mask=None):
    """(n, n_inter, r0, r1, c0, c1) of a boolean image, n_inter against `mask`; an empty box is (2^31 - 1, -1)"""
    image = np.asarray(image, dtype=bool)
    n = int(image.sum())
    ni = 0 if mask is None else int((image & (np.asarray(mask) != 0)).sum())
    if n == 0:
        return n, ni, 2 ** 31 - 1, -1, 2 ** 31 - 1, -1
    rows, cols = np.nonzero(image.any(1))[0], np.nonzero(image.any(0))[0]
    return n, ni, int(rows[0]), int(rows[-1]), int(cols[0]), int(cols[-1])


def _centre(lo, hi):
    return np.float64(lo + hi + 1) * np.float64(0.5)


def _size(lo, hi):
    return np.float64(hi - lo + 1)


def initial_translation(mask, K4, diameter):
    """float64 [3] from one mask [H, W]: z0 = sqrt(fx fy) d / sqrt(w h), x0 = (u - cx) z0 / fx, y0 likewise"""
    n, _, r0, r1, c0, c1 = stats(np.asarray(mask) != 0)
    if n == 0:
        return np.full(3, np.nan)
    fx, fy, cx, cy = (np.float64(v) for v in K4)
    z0 = np.sqrt(fx * fy) * np.float64(diameter) / np.sqrt(_size(c0, c1) * _size(r0, r1))
    return np.array([(_centre(c0, c1) - cx) * z0 / fx, (_centre(r0, r1) - cy) * z0 / fy, z0])


def update(t, sil, msk, K4):
    """one update of t (float64 [3]) from the silhouette's and the mask's stats(); empty -> t unchanged"""
    if sil[0] == 0 or msk[0] == 0:
        return np.array(t, dtype=np.float64)
    fx, fy, cx, cy = (np.float64(v) for v in K4)
    x, y, z = (np.float64(v) for v in t)
    s = np.sqrt((_size(sil[4], sil[5]) * _size(sil[2], sil[3])) / (_size(msk[4], msk[5]) * _size(msk[2], msk[3])))
    z1 = z * s
    pu = fx * x / z + cx
    pv = fy * y / z + cy
    k = z / z1
    u1 = _centre(msk[4], msk[5]) - (_centre(sil[4], sil[5]) - pu) * k
    v1 = _centre(msk[2], msk[3]) - (_centre(sil[2], sil[3]) - pv) * k
    return np.array([(u1 - cx) * z1 / fx, (v1 - cy) * z1 / fy, z1])


def iou(sil, msk):
    """|S n M| / |S u M| from stats(silhouette, mask) and stats(mask); NaN for an empty mask"""
    if msk[0] == 0:
        return np.nan
    return np.float64(sil[1]) / np.float64(sil[0] + msk[0] - sil[1])


def pose(R, t):
    """the rasterizer's float32 [4, 4] pose of [R | t]"""
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T.astype(np.float32)


def cpu_renderer(vertices, faces, K4, image_size, znear=0.05):
    return lambda R, t: ro.render(vertices, faces, pose(R, t), K4, image_size, znear)[0].numpy()


def fit(render, R, t_init, mask, K4, iters):
    """-> (t float64 [3], iou, stats of the silhouette at t) after `iters` updates of one hypothesis"""
    msk = stats(np.asarray(mask) != 0)
    t = np.array(t_init, dtype=np.float64)
    for _ in range(iters):
        t = update(t, stats(render(R, t) > 0, mask), msk, K4)
    sil = stats(render(R, t) > 0, mask)
    if msk[0] == 0:
        return np.full(3, np.nan), np.nan, sil
    return t, iou(sil, msk), sil
