"""Plain-numpy restatement of crop_warp_kernel (nope_b200/csrc/crop.cuh): the reference's input pipeline -- PIL's
paste onto black through a mask, `cv2.warpPerspective` (bilinear, constant border 0) and `ToTensor` + `x*2-1` -- op by
op in the kernel's order.  The GPU tests hold the kernel to this bit for bit; the CPU tests hold this to the live cv2 /
PIL / torchvision pipeline and to tests/golden/crop.npz.  DESIGN.md section 13 states the convention."""
import numpy as np

INTER_BITS = 5
INTER_TAB_SIZE = 1 << INTER_BITS           # 32 sub-pixel steps per pixel
COEF_BITS = 15
COEF_SCALE = 1 << COEF_BITS                # the fixed-point weights sum to 32768
BLOCK_W = 64                               # output columns per coordinate block (S >= 64; S columns when S < 64)
INT_MIN, INT_MAX = -2147483648.0, 2147483647.0


def bilinear_table():
    """int32 [32 * 32, 4]: entry fy * 32 + fx holds the weights of the taps (x, y), (x+1, y), (x, y+1), (x+1, y+1).
    Each weight is the float32 product of the 1-D weights (1 - f, f), f = i * (1/32) in float32, times 32768, rounded
    half to even; when an entry's sum is not 32768 its largest weight (sum short) or smallest weight (sum over) takes
    the difference."""
    scale = np.float32(1.0) / np.float32(INTER_TAB_SIZE)
    one = np.float32(1.0)
    tab1 = [(one - np.float32(i) * scale, np.float32(i) * scale) for i in range(INTER_TAB_SIZE)]
    out = np.zeros((INTER_TAB_SIZE * INTER_TAB_SIZE, 4), dtype=np.int32)
    for i in range(INTER_TAB_SIZE):
        for j in range(INTER_TAB_SIZE):
            w = [int(np.rint(np.float32(tab1[i][k1] * tab1[j][k2]) * np.float32(COEF_SCALE)))
                 for k1 in range(2) for k2 in range(2)]
            diff = sum(w) - COEF_SCALE
            if diff < 0:
                w[int(np.argmax(w))] -= diff
            elif diff > 0:
                w[int(np.argmin(w))] -= diff
            out[i * INTER_TAB_SIZE + j] = w
    return out


def fixed_coords(inv_map, S, block_w=BLOCK_W):
    """inv_map [3, 3] float64 (destination -> source) -> X, Y int32 [S, S], source positions in 1/32 px.  Per output
    pixel (x, y): the block origin xb = x - x % block_w, then X0 = (M0 xb + M1 y) + M2, X = X0 + M0 (x - xb), likewise
    Y and W; W' = 32 / W (0 when W == 0); X W' and Y W' clamped to the int32 range (NaN -> INT_MAX) and rounded half to
    even.  block_w = S gives the naive association ((M0 x + M1 y) + M2)."""
    M = np.asarray(inv_map, dtype=np.float64).reshape(9)
    x = np.arange(S, dtype=np.int64)
    xb = ((x // block_w) * block_w).astype(np.float64)[None, :]
    x1 = (x % block_w).astype(np.float64)[None, :]
    y = np.arange(S, dtype=np.float64)[:, None]
    with np.errstate(all="ignore"):
        X0 = (M[0] * xb + M[1] * y) + M[2]
        Y0 = (M[3] * xb + M[4] * y) + M[5]
        W0 = (M[6] * xb + M[7] * y) + M[8]
        Wd = W0 + M[6] * x1
        Wp = np.where(Wd != 0, np.float64(INTER_TAB_SIZE) / np.where(Wd != 0, Wd, 1.0), 0.0)
        fX = (X0 + M[0] * x1) * Wp
        fY = (Y0 + M[3] * x1) * Wp
    out = []
    for f in (fX, fY):
        f = np.where(f < INT_MAX, f, INT_MAX)              # std::min(INT_MAX, f): NaN -> INT_MAX
        f = np.where(INT_MIN < f, f, INT_MIN)              # std::max(INT_MIN, f)
        out.append(np.rint(f).astype(np.int64).astype(np.int32))
    return out[0], out[1]


def div255(a):
    a = a + 128
    return ((a >> 8) + a) >> 8


def masked_frame(frame, mask=None):
    """uint8 [H, W, 3 | 4] (+ uint8 mask [H, W]) -> int32 [H, W, 3]: PIL's paste of the RGB onto black through the
    mask, DIV255(v m); the alpha channel is the mask of a 4-channel frame, and no mask means m = 255."""
    frame = np.asarray(frame)
    v = frame[..., :3].astype(np.int32)
    if frame.shape[-1] == 4:
        if mask is not None:
            raise ValueError("a 4-channel frame carries its own mask")
        m = frame[..., 3].astype(np.int32)
    elif mask is None:
        return v
    else:
        m = np.asarray(mask).astype(np.int32)
    return div255(v * m[..., None])


def warp_u8(frame, inv_map, S, mask=None, block_w=BLOCK_W):
    """-> uint8 [S, S, 3]: the masked frame warped through inv_map, bilinear from the fixed-point table, taps outside
    the frame 0, (sum v_k w_k + 16384) >> 15 saturated to [0, 255]."""
    src = masked_frame(frame, mask)
    H, W = src.shape[:2]
    X, Y = fixed_coords(inv_map, S, block_w)
    sx, sy = X >> INTER_BITS, Y >> INTER_BITS
    tab = bilinear_table()[(Y & (INTER_TAB_SIZE - 1)) * INTER_TAB_SIZE + (X & (INTER_TAB_SIZE - 1))]   # [S, S, 4]
    acc = np.zeros((S, S, 3), dtype=np.int64)
    for k, (dx, dy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        tx, ty = sx.astype(np.int64) + dx, sy.astype(np.int64) + dy
        inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
        v = src[np.clip(ty, 0, H - 1), np.clip(tx, 0, W - 1)].astype(np.int64)
        acc += np.where(inside[..., None], v, 0) * tab[..., k:k + 1].astype(np.int64)
    return np.clip((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS, 0, 255).astype(np.uint8)


def normalise(u8):
    """uint8 [..., S, S, 3] -> float32 [..., 3, S, S]: ((u / 255) * 2) - 1 in float32, each operation rounded."""
    f = (np.asarray(u8).astype(np.float32) / np.float32(255.0)) * np.float32(2.0) - np.float32(1.0)
    return np.moveaxis(f, -1, -3).astype(np.float32)


def crop(frame, inv_map, S, mask=None):
    """one crop, float32 [3, S, S] in [-1, 1]"""
    return normalise(warp_u8(frame, inv_map, S, mask))


PRIMESENSE_K = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]])   # 720 x 540
SHAPENET_K = np.array([[525.0, 0.0, 256.0], [0.0, 525.0, 256.0], [0.0, 0.0, 1.0]])                    # 512 x 512


def _rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def seeded_cases(n=48, seed=0):
    """n crop cases of uniform-noise frames, cycling S in {256, 64, 17}, the mask (none, binary, graded RGBA alpha),
    keep_inplane, the object's place (inside twice, across the border, outside the frame) and the box's size on
    screen (0.3 S to 3 S px: magnified and minified).  Each: dict(frame uint8 [H, W, 3 | 4], mask uint8 [H, W] or
    None, K, pose [4, 4] (metres), vbs, S, keep_inplane, M (crop_frame's forward map), inv_map, name)."""
    from nope_b200.crop import crop_transforms, forward_map
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n):
        S = (256, 64, 17)[i % 3]
        kind = ("none", "binary", "rgba")[(i // 3) % 3]
        keep_inplane = bool((i // 9) % 2)
        where = ("inside", "inside", "partly", "outside")[(i // 2) % 4]
        K = SHAPENET_K if kind == "rgba" else PRIMESENSE_K
        H, W = (512, 512) if kind == "rgba" else (540, 720)
        if i % 5 == 4:                                      # an odd-sized frame with its own intrinsics
            H, W = 251, 333
            K = np.array([[300.0, 0.0, 166.4], [0.0, 310.0, 125.1], [0.0, 0.0, 1.0]])
        Z = rng.uniform(0.4, 1.6)
        box_px = S * np.exp(rng.uniform(np.log(0.3), np.log(3.0)))
        vbs = box_px * Z / K[0, 0]
        if where == "inside":
            u, v = rng.uniform(0.2 * W, 0.8 * W), rng.uniform(0.2 * H, 0.8 * H)
        elif where == "partly":
            u, v = rng.choice([0.0, W]) + rng.uniform(-0.3, 0.3) * box_px, rng.uniform(0, H)
        else:
            u, v = W + 1.5 * box_px + 10, rng.uniform(-H, 2 * H)
        pose = np.eye(4)
        pose[:3, :3] = _rotation(rng)
        pose[:3, 3] = [(u - K[0, 2]) * Z / K[0, 0], (v - K[1, 2]) * Z / K[1, 1], Z]
        frame = rng.integers(0, 256, (H, W, 4 if kind == "rgba" else 3), dtype=np.uint8)
        mask = None
        if kind == "binary":
            mask = (rng.random((H, W)) < 0.7).astype(np.uint8) * 255
        elif kind == "rgba" and i % 2:
            frame[..., 3] = np.where(rng.random((H, W)) < 0.2, 0, 255)       # binary alpha besides graded
        M = forward_map(K, pose, vbs, S, keep_inplane)
        inv = crop_transforms(K, pose, vbs, S, keep_inplane)[0]
        cases.append(dict(frame=frame, mask=mask, K=K, pose=pose, vbs=vbs, S=S, keep_inplane=keep_inplane, M=M,
                          inv_map=inv, name=f"{i}:{kind}/{where}/S{S}/{'inplane' if keep_inplane else 'upright'}/"
                                            f"{H}x{W}/{box_px / S:.2f}S"))
    return cases


def crop_frames(frames, inv_maps, S, masks=None, frame_idx=None):
    """The batched call of nope_crop_frames: frames [F, H, W, C], inv_maps [B, 3, 3], masks [B, H, W] or None,
    frame_idx [B] or None (then F == B) -> float32 [B, 3, S, S]; a frame index outside [0, F) gives -1 everywhere."""
    frames = np.asarray(frames)
    inv_maps = np.asarray(inv_maps, dtype=np.float64).reshape(-1, 3, 3)
    B = len(inv_maps)
    idx = np.arange(B) if frame_idx is None else np.asarray(frame_idx)
    out = np.full((B, 3, S, S), -1.0, dtype=np.float32)
    for b in range(B):
        if 0 <= idx[b] < len(frames):
            out[b] = crop(frames[idx[b]], inv_maps[b], S, None if masks is None else masks[b])
    return out
