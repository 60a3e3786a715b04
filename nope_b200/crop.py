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
            _lib.stream(dev)))
    return out


# ------------------------------------------------------------------ the crop camera (DESIGN.md section 23)
MAX_CAMERAS = 65535      # F (poses, detections) and P (rotations per pose) of nope_crop_camera / nope_crop_rotate



def _camera(pose, keep_inplane, dev):
    """R_v float64 [F, 3, 3] on `dev` of host poses float64 [F, 4, 4]; the pose is checked here and staged by the
    library in stream order: no synchronisation"""
    F_ = pose.shape[0]
    if F_ > MAX_CAMERAS:
        raise ValueError(f"at most {MAX_CAMERAS} poses, got {F_}")
    read = pose[:, :3, 3] if keep_inplane else pose[:, :3]
    if not np.isfinite(read).all():
        raise ValueError("pose must be finite")
    if keep_inplane and not (pose[:, 2, 3] > 0).all():
        raise ValueError("keep_inplane needs every object centre in front of the camera (Z > 0)")
    host = np.ascontiguousarray(pose, dtype=np.float64)
    with torch.cuda.device(dev):
        out = torch.empty((F_, 3, 3), device=dev, dtype=torch.float64)
        _lib.check(_lib.load().nope_crop_camera(C.c_void_p(host.ctypes.data), F_, int(bool(keep_inplane)),
                                                _lib.ptr(out), _lib.stream(dev)))
    return out


def crop_camera(pose, keep_inplane=True):
    """The crop camera's rotation R_v float64 [F, 3, 3] (or [3, 3] for one pose) of the crops `crop_transforms` cuts
    around pose [F, 4, 4] or [4, 4] (object -> OpenCV camera): a crop is the view of a pinhole camera at the real
    camera's centre, with rotation R_v and intrinsics `crop_intrinsics`, so a rotation R in the real camera is
    R_v R in the crop's (`to_crop`, `to_camera`).  keep_inplane as crop_transforms: True reads the translation only
    (Z > 0), False the top three rows.  The pose must be a CUDA tensor (there is no CPU fallback); it is read on the
    host, one device -> host copy, because the library checks every pose before it launches.  ValueError for a
    malformed or non-finite pose, NopeError for a host one."""
    if not torch.is_tensor(pose) or pose.device.type != "cuda":
        raise _lib.NopeError("crop_camera needs a CUDA pose tensor (no CPU fallback)")
    one = pose.dim() == 2
    P = _batched(pose.detach().to("cpu", torch.float64).numpy(), (4, 4), "pose")
    out = _camera(P, keep_inplane, pose.device)
    return out[0] if one else out


def crop_intrinsics(pose, virtual_bbox_size, image_size=256):
    """The crop camera's intrinsics K_v float64 [F, 3, 3] (or [3, 3] for one pose) of the crops `crop_transforms`
    cuts around pose [F, 4, 4] or [4, 4] with side virtual_bbox_size (a number or [F], the pose's units) and crop
    side S = image_size: f_v = S |o| / s and the principal point (S/2, S/2), o = pose[:3, 3].  Plain torch on the
    pose's device.  Exact up to the int32 truncation of crop_frame's corners, and not in crop_frame's image-axes
    fallback (crop_camera's R_v = I), whose square is not perpendicular to o."""
    from .translation import _sqrt
    p = _tensor(pose).to(torch.float64)
    one = p.dim() == 2
    p = p[None] if one else p
    if p.dim() != 3 or p.shape[1:] != (4, 4):
        raise ValueError(f"pose [4, 4] or [F, 4, 4] expected, got {list(p.shape)}")
    S = int(image_size)
    if S != image_size or not 1 <= S <= MAX_CROP:
        raise ValueError(f"image_size must be an integer in [1, {MAX_CROP}], got {image_size!r}")
    s = _tensor(virtual_bbox_size).to(device=p.device, dtype=torch.float64).reshape(-1)
    if s.shape[0] not in (1, p.shape[0]):
        raise ValueError(f"virtual_bbox_size: a number or [F] with F = {p.shape[0]} expected, got {list(s.shape)}")
    o = p[:, :3, 3]
    norm = _sqrt((o[:, 0] * o[:, 0] + o[:, 1] * o[:, 1]) + o[:, 2] * o[:, 2])
    K = torch.zeros((p.shape[0], 3, 3), dtype=torch.float64, device=p.device)
    K[:, 0, 0] = K[:, 1, 1] = S * norm / s
    K[:, 0, 2] = K[:, 1, 2] = S / 2
    K[:, 2, 2] = 1.0
    return K[0] if one else K


def _rotate(R, Rv, to_camera, name):
    if not (torch.is_tensor(R) and torch.is_tensor(Rv)) or R.device.type != "cuda" or Rv.device != R.device:
        raise _lib.NopeError(f"{name} needs R and Rv as CUDA tensors on one device (no CPU fallback)")
    if R.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"R must be float32 or float64, got {R.dtype}")
    if R.dim() not in (3, 4) or R.shape[-2:] != (3, 3) or Rv.shape != (R.shape[0], 3, 3) or R.shape[0] < 1 or \
            (R.dim() == 4 and R.shape[1] < 1):
        raise ValueError(f"R [F, P, 3, 3] or [F, 3, 3] and Rv [F, 3, 3] expected, got {list(R.shape)} and "
                         f"{list(Rv.shape)}")
    F_, P = R.shape[0], (R.shape[1] if R.dim() == 4 else 1)
    if F_ > MAX_CAMERAS or P > MAX_CAMERAS:
        raise ValueError(f"F and P must be at most {MAX_CAMERAS}, got {F_} and {P}")
    if Rv.dtype != torch.float64:
        raise ValueError(f"Rv must be float64 (crop_camera's), got {Rv.dtype}")
    dev = R.device
    with torch.cuda.device(dev):
        src = R.detach().to(torch.float64).contiguous()
        out = torch.empty_like(src)
        _lib.check(_lib.load().nope_crop_rotate(_lib.ptr(Rv.contiguous()), F_, _lib.ptr(src), P, int(to_camera),
                                                _lib.ptr(out), _lib.stream(dev)))
    return out


def to_camera(R_crop, Rv):
    """A rotation in the crop's camera re-expressed in the real camera: R_v^T R_crop, float64 in R_crop's shape
    ([F, P, 3, 3] or [F, 3, 3], float32 or float64) on its CUDA device; Rv [F, 3, 3] from crop_camera.  Runs on the
    current stream without synchronising."""
    return _rotate(R_crop, Rv, True, "to_camera")


def to_crop(R_cam, Rv):
    """A rotation in the real camera expressed in the crop's camera: R_v R_cam; shapes and devices as to_camera.
    For a reference cut from a real frame, its pose's rotation in its crop's camera, e.g. for
    poses.relative_rotation_6d."""
    return _rotate(R_cam, Rv, False, "to_crop")


def frame_crops(frames, masks, K, diameter, image_size=256, frame_idx=None, bbox_scale=1.2):
    """Crops of B detections in camera frames for the pose searches, and the crop cameras that map the searches'
    rotations back to the frames (DESIGN.md section 23):
      frames     uint8 [F, H, W, 3] RGB (host or CUDA; the crops go to the frames' CUDA device, or the current one)
      masks      uint8 or bool [B, H, W], one per detection, nonzero = object (host or on the frames' device); a
                 uint8 mask is pasted as crop_frames pastes it (a BOP mask_visib is 0 / 255), a bool one as 0 / 255
      K          [3, 3] or [B, 3, 3] intrinsics, read on the host (host data saves a copy)
      diameter   the object diameter, a number or [B] (mm)
      frame_idx  integer [B], or None when F == B: the frame of each detection
      bbox_scale the crop's square is bbox_scale * diameter wide (1.2, as src/dataloader/bop.py:193-194)
    It runs `translation.initial_translation` on the masks' device (t0 [B, 3], mm), `crop_transforms(K, t0,
    bbox_scale * diameter, keep_inplane=True)` on the host, `crop_frames` and `crop_camera`.
    -> (crops float32 [B, 3, S, S], t0 float64 [B, 3] on the masks' device, R_v float64 [B, 3, 3] on the crops'
    device, inv_maps float64 [B, 3, 3] on the host).  The one host synchronisation is the copy of t0 that the host
    geometry needs (none for host masks).  ValueError for an empty mask or a malformed argument."""
    from .translation import initial_translation
    m = _tensor(masks)
    if m.dim() != 3 or m.shape[0] < 1 or m.dtype not in (torch.uint8, torch.bool):
        raise ValueError(f"masks must be uint8 or bool [B, H, W], got {m.dtype} {list(m.shape)}")
    B = m.shape[0]
    Kh = _batched(_as_numpy(K, "K"), (3, 3), "K")
    if len(Kh) not in (1, B):
        raise ValueError(f"K [3, 3] or [B, 3, 3] with B = {B} expected, got {list(Kh.shape)}")
    Kh = np.ascontiguousarray(np.broadcast_to(Kh, (B, 3, 3)))
    d = _as_numpy(diameter, "diameter").reshape(-1)
    if len(d) not in (1, B) or not (np.isfinite(d).all() and (d > 0).all()):
        raise ValueError(f"diameter: a finite number > 0 or [B] with B = {B} expected, got {d.tolist()}")
    t0 = initial_translation(m, torch.from_numpy(Kh), torch.from_numpy(np.broadcast_to(d, (B,)).copy()))
    th = t0.cpu().numpy()                                   # the host geometry's one copy
    bad = np.flatnonzero(~np.isfinite(th).all(1))
    if len(bad):
        raise ValueError(f"detections {bad.tolist()} have an empty mask")
    pose = np.tile(np.eye(4), (B, 1, 1))
    pose[:, :3, 3] = th
    inv_maps = crop_transforms(Kh, pose, bbox_scale * d, image_size, keep_inplane=True)
    fr = _tensor(frames)
    if fr.dim() != 4 or fr.shape[3] != 3:
        raise ValueError(f"frames must be uint8 [F, H, W, 3], got {fr.dtype} {list(fr.shape)}")
    dev = fr.device if fr.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    paste = m.to(torch.uint8) * 255 if m.dtype == torch.bool else m
    crops = crop_frames(fr, torch.from_numpy(inv_maps), image_size, masks=paste, frame_idx=frame_idx)
    Rv = _camera(pose, True, dev)
    return crops, t0, Rv, torch.from_numpy(inv_maps)


def detection_occluders(masks, frame_idx=None, num_frames=None):
    """The occluders of B detections that share frames (DESIGN.md section 24): O_b = (the union of the masks of the
    other detections of frame frame_idx[b]) minus b's own mask, uint8 [B, H, W] (1 = another detection may hide the
    object there) on the masks' device.
      masks      uint8 or bool [B, H, W], one per detection, nonzero = object (host or CUDA)
      frame_idx  integer [B] (host or on the masks' device), or None for one frame per detection (every O_b empty)
      num_frames F, the number of frames; indices outside [0, F) share one group below 0 and one at F or above (they
                 are crop_frames' all-black crops).  None: max(frame_idx) + 1, read on the host.
    A per-frame count of the masks (`index_add_`) minus the detection's own: plain torch, no host synchronisation for
    host frame indices or a given num_frames."""
    m = _tensor(masks)
    if m.dim() != 3 or m.shape[0] < 1 or m.dtype not in (torch.uint8, torch.bool):
        raise ValueError(f"masks must be uint8 or bool [B, H, W], got {m.dtype} {list(m.shape)}")
    B = m.shape[0]
    if frame_idx is None:
        fi, F_ = torch.arange(B), B
    else:
        fi = _tensor(frame_idx)
        if fi.is_floating_point() or fi.is_complex() or fi.dtype == torch.bool or tuple(fi.shape) != (B,):
            raise ValueError(f"frame_idx must be integer [B] = [{B}], got {fi.dtype} {list(fi.shape)}")
        F_ = int(fi.max()) + 1 if num_frames is None else int(num_frames)
    if F_ < 1:
        raise ValueError(f"num_frames must be >= 1, got {F_}")
    from .bop import _to_dev
    fi = _to_dev(fi, m.device, torch.int64).clamp(-1, F_) + 1              # groups 0 ... F + 1
    own = (m != 0).to(torch.int32)
    count = torch.zeros((F_ + 2,) + tuple(m.shape[1:]), dtype=torch.int32, device=m.device).index_add_(0, fi, own)
    return ((count[fi] > own) & (own == 0)).to(torch.uint8)
