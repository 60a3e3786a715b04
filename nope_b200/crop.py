"""Full-frame crops on the GPU (DESIGN.md section 13): the reference's virtual-bounding-box crop (`crop_frame`,
src/poses/utils.py:204-272) with the input pipeline of its dataloaders around it -- PIL's paste onto black through the
object mask, `cv2.warpPerspective` (bilinear, constant border 0), `ToTensor` / `Resize(S)` / `x*2-1`
(src/dataloader/bop.py:111-117, 188-226; shapeNet.py:64-70, 167-210).  `crop_transforms` is the host geometry,
`crop_frames` the CUDA warp (crop.cuh); the crops equal the reference's bit for bit.  There is no CPU fallback."""
import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_SIDE = 16384          # frame H, W
MAX_CROP = 4096           # crop side S


def _as_numpy(x, name):
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    try:
        return np.asarray(x, dtype=np.float64)
    except (TypeError, ValueError) as exc:
        raise ValueError(f"{name} must be numeric") from exc


def _batched(x, tail, name):
    if x.shape == tail:
        return x[None]
    if x.ndim == len(tail) + 1 and x.shape[1:] == tail and x.shape[0] >= 1:
        return x
    raise ValueError(f"{name} {list(tail)} or [B, {', '.join(map(str, tail))}] expected, got {list(x.shape)}")


def _corners(intrinsic, pose, virtual_bbox_size, keep_inplane):
    """crop_frame's four projected corners (utils.py:213-258), int32 [4, 2]: w1 = c + up - right, w2 = c - up - right,
    w3 = c + up + right, w4 = c - up + right, each projected with `perspective` (utils.py:50-57) and truncated."""
    origin_in_cam = np.dot(pose, np.array([0, 0, 0, 1.0]))[0:3]
    if not origin_in_cam[2] > 0:
        raise ValueError(f"the object centre must lie in front of the camera (Z > 0), got Z = {origin_in_cam[2]}")
    o = origin_in_cam
    if keep_inplane:
        upper = np.array([0.0, -o[2], o[1]])
        right = np.array([o[1] * o[1] + o[2] * o[2], -o[0] * o[1], -o[0] * o[2]])
    else:
        # the world's "up" at Z = 6 (metres, as the BOP loaders convert), taken through the pose
        up = np.array([0, 0, 6]) - o
        up = np.dot(pose, [up[0], up[1], up[2], 1])[0:3]
        right = np.cross(o, up)
        upper = np.cross(right, o)
    if np.linalg.norm(upper) == 0 and np.linalg.norm(right) == 0:
        # both branches fall back to the image axes; with keep_inplane this needs Z = 0, refused above
        upper = np.array([0, -1, 0])
        right = np.array([1, 0, 0])
    upper = upper * (virtual_bbox_size / 2) / np.linalg.norm(upper)
    right = right * (virtual_bbox_size / 2) / np.linalg.norm(right)
    pts = [o + upper - right, o - upper - right, o + upper + right, o - upper + right]
    eye = np.eye(4)
    R, T = eye[:3, :3], eye[:3, 3]
    out = np.zeros((4, 2))
    for i, p in enumerate(pts):
        rep = np.matmul(intrinsic, np.matmul(R, p.reshape(3, 1)) + T.reshape(3, 1))
        with np.errstate(all="ignore"):
            uv = (rep[0] / rep[2], rep[1] / rep[2])
        for j, q in enumerate(uv):
            if not (np.isfinite(q).all() and -2147483648.0 < q[0] < 2147483648.0):
                raise ValueError(f"corner {i + 1} of the virtual box projects to {q[0]}, outside the int32 range")
            out[i, j] = np.int32(q[0])
    return out.astype(np.int32)


def crop_transforms(intrinsic, pose, virtual_bbox_size, image_size=256, keep_inplane=False):
    """Destination -> source maps float64 [B, 3, 3] of the reference's virtual-bounding-box crop, computed on the host:
    the `M` that `crop_frame` (src/poses/utils.py:204-264) hands `cv2.warpPerspective`, inverted as warpPerspective
    inverts it (`cv2.invert`, DECOMP_LU).

      intrinsic          [3, 3] or [B, 3, 3] pixels (shapeNet.py:172, bop.py:227)
      pose               [4, 4] or [B, 4, 4] object -> OpenCV camera; only its translation is used when keep_inplane
      virtual_bbox_size  scalar or [B], the side of the square around the object centre, in the pose's units
      image_size         S, the side of the crop
      keep_inplane       crop_frame's flag: False aligns the crop's "up" with the world's, True keeps the roll

    The keep_inplane=False rule mixes the translation with a constant 6, so it expects metres, as bop.py:196-199
    converts (pose[:3, 3] / 1000 and diameter * 1.2 / 1000).  Raises ValueError for malformed shapes, an object centre
    at Z <= 0 or a map that is not finite."""
    import cv2

    K = _as_numpy(intrinsic, "intrinsic")
    P = _as_numpy(pose, "pose")
    V = _as_numpy(virtual_bbox_size, "virtual_bbox_size")
    K, P = _batched(K, (3, 3), "intrinsic"), _batched(P, (4, 4), "pose")
    if V.ndim > 1:
        raise ValueError(f"virtual_bbox_size must be a scalar or [B], got {list(V.shape)}")
    V = V.reshape(-1)
    S = int(image_size)
    if S != image_size or not 1 <= S <= MAX_CROP:
        raise ValueError(f"image_size must be an integer in [1, {MAX_CROP}], got {image_size!r}")
    B = max(len(K), len(P), len(V))
    for x, name in ((K, "intrinsic"), (P, "pose"), (V, "virtual_bbox_size")):
        if len(x) not in (1, B):
            raise ValueError(f"{name} has batch size {len(x)}, expected 1 or {B}")
    if not (np.isfinite(V).all() and (V > 0).all()):
        raise ValueError("virtual_bbox_size must be finite and > 0")
    out = np.empty((B, 3, 3), dtype=np.float64)
    for b in range(B):
        M = forward_map(K[b % len(K)], P[b % len(P)], float(V[b % len(V)]), S, keep_inplane)
        _, out[b] = cv2.invert(M, flags=cv2.DECOMP_LU)
        if not np.isfinite(out[b]).all():
            raise ValueError(f"crop {b}: the perspective map is not finite")
    return out


def forward_map(intrinsic, pose, virtual_bbox_size, image_size, keep_inplane=False):
    """The source -> destination `M` of one crop, as crop_frame hands it to cv2.warpPerspective (utils.py:257-265):
    the truncated corners onto [[0, 0], [0, 1], [1, 0], [1, 1]] * S by cv2.getPerspectiveTransform.  intrinsic [3, 3]
    and pose [4, 4] float64; crop_transforms checks the arguments and inverts this."""
    import cv2

    corners = _corners(intrinsic, pose, virtual_bbox_size, keep_inplane)
    target = np.array([[0, 0], [0, 1], [1, 0], [1, 1]]).astype(np.float32) * image_size
    return cv2.getPerspectiveTransform(corners.astype(np.float32), target)


def _to_device(dev, t):
    """host tensors travel through pinned memory, once"""
    if t.device.type == "cpu":
        return t.contiguous().pin_memory().to(dev, non_blocking=True)
    return t.contiguous()


def _tensor(x):
    return x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))


def crop_frames(frames, inv_maps, image_size=256, masks=None, frame_idx=None):
    """Crops float32 [B, 3, S, S] in [-1, 1] on the frames' CUDA device (the current one for host frames): crop b
    warps frame frame_idx[b] through inv_maps[b] as the reference's dataloaders build their inputs --
    `black.paste(rgb, mask)` (bop.py:223-225, shapeNet.py:206-208), `cv2.warpPerspective(img, M, (S, S))` with
    M^-1 = inv_maps[b] (utils.py:265), then `ToTensor` / `Resize(S)` / `x*2-1` (bop.py:111-117).

      frames     uint8 [F, H, W, 3] RGB or [F, H, W, 4] RGBA (the alpha is the mask), 1 <= H, W <= 16384
      inv_maps   float64 [B, 3, 3] or [B, 9], from crop_transforms
      image_size S, 1 <= S <= 4096
      masks      uint8 [B, H, W], one per crop (a BOP mask_visib belongs to one instance), or None (all 255)
      frame_idx  integer [B], or None when F == B; an index outside [0, F) gives an all-black crop (-1)

    Host inputs are uploaded once through pinned memory; device inputs must be on the frames' device.  Argument errors
    raise before any device work; the call runs on the current stream and does not synchronise."""
    frames, inv_maps = _tensor(frames), _tensor(inv_maps)
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] not in (3, 4):
        raise ValueError(f"frames must be uint8 [F, H, W, 3 | 4], got {frames.dtype} {list(frames.shape)}")
    F_, H, W, Cn = frames.shape
    if F_ < 1 or not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"frames need F >= 1 and H, W in [1, {MAX_SIDE}], got {list(frames.shape)}")
    S = int(image_size)
    if S != image_size or not 1 <= S <= MAX_CROP:
        raise ValueError(f"image_size must be an integer in [1, {MAX_CROP}], got {image_size!r}")
    if inv_maps.dtype != torch.float64:
        raise ValueError(f"inv_maps must be float64, got {inv_maps.dtype}")
    if inv_maps.dim() == 2 and inv_maps.shape[1] == 9:
        inv_maps = inv_maps.reshape(-1, 3, 3)
    if inv_maps.dim() != 3 or inv_maps.shape[1:] != (3, 3) or inv_maps.shape[0] < 1:
        raise ValueError(f"inv_maps [B, 3, 3] or [B, 9] expected, got {list(inv_maps.shape)}")
    B = inv_maps.shape[0]
    if masks is not None:
        masks = _tensor(masks)
        if Cn == 4:
            raise ValueError("RGBA frames carry their mask in the alpha channel: pass masks=None")
        if masks.dtype != torch.uint8 or tuple(masks.shape) != (B, H, W):
            raise ValueError(f"masks must be uint8 [B, H, W] = {[B, H, W]}, got {masks.dtype} {list(masks.shape)}")
    if frame_idx is None:
        if F_ != B:
            raise ValueError(f"without frame_idx there must be one frame per crop: F = {F_}, B = {B}")
    else:
        frame_idx = _tensor(frame_idx)
        if frame_idx.is_floating_point() or frame_idx.is_complex() or frame_idx.dtype == torch.bool or \
                tuple(frame_idx.shape) != (B,):
            raise ValueError(f"frame_idx must be integer [B] = [{B}], got {frame_idx.dtype} {list(frame_idx.shape)}")
        if frame_idx.device.type == "cpu":
            # an index outside [0, F) is a black crop: keep it outside after the narrowing to int32
            frame_idx = frame_idx.to(torch.int64).clamp(-1, F_).to(torch.int32)
    dev = frames.device if frames.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    for t, name in ((inv_maps, "inv_maps"), (masks, "masks"), (frame_idx, "frame_idx")):
        if t is not None and t.device.type != "cpu" and t.device != dev:
            raise ValueError(f"{name} is on {t.device}, the frames on {dev}")
    with torch.cuda.device(dev):
        fr = _to_device(dev, frames)
        mp = _to_device(dev, inv_maps)
        mk = None if masks is None else _to_device(dev, masks)
        fi = None if frame_idx is None else _to_device(dev, frame_idx).to(torch.int32)
        out = torch.empty((B, 3, S, S), device=dev, dtype=torch.float32)
        _lib.check(_lib.load().nope_crop_frames(
            _lib.ptr(fr), F_, H, W, Cn, _lib.ptr(mk), _lib.ptr(fi), _lib.ptr(mp), B, S, _lib.ptr(out),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out
