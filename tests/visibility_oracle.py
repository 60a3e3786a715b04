"""Plain-numpy restatement of the searches under occlusion (DESIGN.md section 27): crop_hidden_kernel with the crop
warp's own fixed-point sample (oracle/crop_oracle.py), latent_visibility_kernel with the roll's float32 sample in
inplane_rotate_kernel's order (oracle/inplane_oracle.py), and the float64 scores over the visible latent pixels.
The GPU tests hold the kernels to the first two bit for bit."""
import numpy as np

from oracle import crop_oracle

LATENT = 32


def crop_hidden(occluders, inv_maps, S=256):
    """occluders [B, H, W] (non-zero = may be hidden), inv_maps [B, 3, 3] float64 -> uint8 [B, S, S]: 1 where a tap
    of the crop warp's sample has a non-zero fixed-point weight, lies inside the frame and is occluded."""
    occ = np.asarray(occluders) != 0
    maps = np.asarray(inv_maps, dtype=np.float64).reshape(-1, 3, 3)
    B, H, W = occ.shape
    tab = crop_oracle.bilinear_table()
    out = np.zeros((B, S, S), dtype=np.uint8)
    for b in range(B):
        X, Y = crop_oracle.fixed_coords(maps[b], S)
        sx, sy = (X >> crop_oracle.INTER_BITS).astype(np.int64), (Y >> crop_oracle.INTER_BITS).astype(np.int64)
        wt = tab[(Y & 31) * 32 + (X & 31)]                                                   # [S, S, 4]
        hid = np.zeros((S, S), dtype=bool)
        for k, (dx, dy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
            tx, ty = sx + dx, sy + dy
            inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
            hid |= (wt[..., k] != 0) & inside & occ[b][np.clip(ty, 0, H - 1), np.clip(tx, 0, W - 1)]
        out[b] = hid
    return out


def roll_sample(c, s, S):
    """inplane_rotate_kernel's sample of every pixel of a copy rolled by (c, s) (float32, one rounding per operation,
    oracle/inplane_oracle.rotate's order) -> (ix, iy int64, fx, fy float32) [S, S]"""
    f32 = np.float32
    c, s = f32(c), f32(s)
    cx = f32(S - 1) * f32(0.5)
    dx = (np.arange(S, dtype=f32) - cx)[None, :]
    dy = (np.arange(S, dtype=f32) - cx)[:, None]
    sx = (c * dx - s * dy) + cx
    sy = (s * dx + c * dy) + cx
    x0, y0 = np.floor(sx), np.floor(sy)
    return x0.astype(np.int64), y0.astype(np.int64), (sx - x0).astype(f32), (sy - y0).astype(f32)


def rolled_hidden(hidden, c, s):
    """Hr [S, S] bool: a tap (ix, iy), (ix + 1, iy) if fx > 0, (ix, iy + 1) if fy > 0, (ix + 1, iy + 1) if both, inside
    the image and hidden"""
    hid = np.asarray(hidden) != 0
    S = hid.shape[0]
    ix, iy, fx, fy = roll_sample(c, s, S)
    out = np.zeros((S, S), dtype=bool)
    for ddx, ddy, use in ((0, 0, np.ones_like(fx, bool)), (1, 0, fx > 0), (0, 1, fy > 0), (1, 1, (fx > 0) & (fy > 0))):
        tx, ty = ix + ddx, iy + ddy
        inside = (tx >= 0) & (tx < S) & (ty >= 0) & (ty < S)
        out |= use & inside & hid[np.clip(ty, 0, S - 1), np.clip(tx, 0, S - 1)]
    return out


def block_visible(hr):
    """Hr [S, S] -> V [32, 32] uint8: 0 where the 8 x 8 block holds a hidden pixel"""
    S = hr.shape[0]
    blk = S // LATENT
    return (~hr.reshape(LATENT, blk, LATENT, blk).any(axis=(1, 3))).astype(np.uint8)


def latent_visibility(hidden, image_idx, cossin):
    """hidden [B, S, S], pairs image_idx [P], cossin [P, 2] float32 -> uint8 [P, 32, 32]; an image index outside
    [0, B) gives an all-visible row"""
    hidden = np.asarray(hidden)
    cossin = np.asarray(cossin, dtype=np.float32)
    out = np.ones((len(image_idx), LATENT, LATENT), dtype=np.uint8)
    for p, b in enumerate(np.asarray(image_idx)):
        if 0 <= b < hidden.shape[0]:
            out[p] = block_visible(rolled_hidden(hidden[b], cossin[p, 0], cossin[p, 1]))
    return out


def scores(query, templates, visible, metric="l2", threshold=0.2):
    """float64 scores of section 27: query [C, hw], templates [N, C, hw], visible [hw] -> [N]; NaN when no pixel is
    visible"""
    q = np.asarray(query, dtype=np.float64)
    t = np.asarray(templates, dtype=np.float64)
    v = np.asarray(visible).reshape(-1) != 0
    n, hw = int(v.sum()), v.size
    if n == 0:
        return np.full(t.shape[0], np.nan)
    q, t = q[:, v], t[:, :, v]
    if metric == "l2":
        return -np.sqrt(((q[None] - t) ** 4).sum(axis=1)).sum(axis=1) * (hw / n)
    if metric == "cosine":
        num = (q[None] * t).sum(axis=(1, 2))
        return num / (np.maximum(np.sqrt((q * q).sum()), 1e-8) * np.maximum(np.sqrt((t * t).sum(axis=(1, 2))), 1e-8))
    per = (q[None] * t).sum(axis=1) / (np.maximum(np.sqrt((q * q).sum(axis=0)), 1e-8)[None]
                                       * np.maximum(np.sqrt((t * t).sum(axis=1)), 1e-8))
    return np.where(per > threshold, per, 0.0).sum(axis=1) / n
