"""Translation from the object mask (DESIGN.md section 18).  Every search of this project returns a rotation; this
module fits, for each frame and rotation hypothesis, the translation whose rendered silhouette lines up with the
object's mask in the frame, and reports the silhouette IoU there.

`initial_translation` is a rotation-agnostic start from the mask's bounding box and the object diameter (plain torch,
CPU or GPU).  `estimate_translation` runs the fit on the GPU (`nope_fit_translation_occluded`,
csrc/translation.cuh): each update renders the silhouette with the depth rasterizer of `nope_b200.vsd`, scales the
distance by the ratio of the bounding-box sizes and moves the origin so the silhouette's box centre lands on the
mask's.  There is no CPU fallback.
A mask cut by the frame border has a cut bounding box, and the fit follows it: no special handling."""
import numpy as np
import torch

from . import _lib
from ._posefit import _masks, _tensor, broadcast_t, cuda_device, fit_args, workspace
from .bop import _to_dev

DEFAULT_ITERS = 4            # from the convergence table of DESIGN.md section 18


def _k4(K, F, device):
    """K [F, 3, 3], [F, 4], [3, 3] or [4] -> float64 [F, 4] (fx, fy, cx, cy) on `device`, without synchronising"""
    k = _tensor(K)
    if k.shape in ((3, 3), (4,)):
        k = k[None]
    if k.dim() == 3 and k.shape[1:] == (3, 3):
        k = torch.stack([k[:, 0, 0], k[:, 1, 1], k[:, 0, 2], k[:, 1, 2]], dim=1)
    if k.dim() != 2 or k.shape[1] != 4 or k.shape[0] not in (1, F):
        raise ValueError(f"K [F, 3, 3] or [F, 4] with F = {F} expected, got {tuple(k.shape)}")
    k = k.to(torch.float64)
    if k.device.type == "cpu" and device.type == "cuda":
        k = k.contiguous().pin_memory().to(device, non_blocking=True)
    return k.to(device).expand(F, 4)


def _sqrt(x):
    """correctly rounded float64 square root: torch's CUDA sqrt is; its vectorised CPU sqrt is not (sqrt(2) comes out
    one ulp off), so host tensors go through numpy's"""
    return torch.sqrt(x) if x.device.type != "cpu" else torch.from_numpy(np.sqrt(x.numpy()))


def mask_box(masks):
    """Integer statistics of masks [F, H, W] (nonzero = object): -> (n, r0, r1, c0, c1), int64 [F] each, on the
    masks' device without synchronising; the box of an empty mask is r0 = H, r1 = -1, c0 = W, c1 = -1."""
    m = _masks(masks) != 0
    F, H, W = m.shape
    rows, cols = m.any(2), m.any(1)
    ar, ac = torch.arange(H, device=m.device), torch.arange(W, device=m.device)
    r0 = torch.where(rows, ar, H).amin(1)
    r1 = torch.where(rows, ar, -1).amax(1)
    c0 = torch.where(cols, ac, W).amin(1)
    c1 = torch.where(cols, ac, -1).amax(1)
    return m.sum((1, 2)), r0, r1, c0, c1


def initial_translation(masks, K, diameter):
    """Rotation-agnostic translation float64 [F, 3] (mm, OpenCV camera) from each frame's mask [F, H, W] (uint8 or
    bool, nonzero = object), intrinsics K [F, 3, 3] or [F, 4] and the object diameter (mm; a number or [F]):
      z0 = sqrt(fx fy) d / sqrt(w h),  x0 = (u - cx) z0 / fx,  y0 = (v - cy) z0 / fy,
    with the mask's box centre u = (c0 + c1 + 1) / 2, v = (r0 + r1 + 1) / 2 and size w = c1 - c0 + 1, h = r1 - r0 + 1
    (pixel (r, c) samples the image point (c + 1/2, r + 1/2)).  NaN for an empty mask.  Plain torch on the masks'
    device, every operation rounded on its own; no synchronisation.  It takes no occluders: under occlusion it starts
    from the visible mask's box, and `estimate_translation(..., occluders=)` corrects from there (DESIGN.md
    section 24)."""
    n, r0, r1, c0, c1 = mask_box(masks)
    dev = n.device
    F = n.shape[0]
    k = _k4(K, F, dev)
    d = _tensor(diameter).to(torch.float64)
    if d.dim() > 1 or (d.dim() == 1 and d.shape[0] not in (1, F)):
        raise ValueError(f"diameter: a number or [F] with F = {F} expected, got {tuple(d.shape)}")
    d = _to_dev(d, dev, torch.float64).expand(F)                  # a host number: pinned, no synchronisation
    fx, fy, cx, cy = k[:, 0], k[:, 1], k[:, 2], k[:, 3]
    w, h = (c1 - c0 + 1).to(torch.float64), (r1 - r0 + 1).to(torch.float64)
    u, v = (c0 + c1 + 1).to(torch.float64) * 0.5, (r0 + r1 + 1).to(torch.float64) * 0.5
    z0 = _sqrt(fx * fy) * d / _sqrt(w * h)
    x0 = (u - cx) * z0 / fx
    y0 = (v - cy) * z0 / fy
    t = torch.stack([x0, y0, z0], dim=1)
    return torch.where((n > 0)[:, None], t, torch.full_like(t, float("nan")))


def occluder_masks(occluders, masks):
    """occluders [F, H, W] (or [H, W] for F = 1; uint8 or bool, nonzero = something may hide the object) checked
    against masks [F, H, W]: -> the occluders as `_masks` returns them, None for None"""
    if occluders is None:
        return None
    o = _masks(occluders)
    if o.shape != masks.shape:
        raise ValueError(f"occluders {tuple(masks.shape)} (the masks' shape) expected, got {tuple(o.shape)}")
    return o


def estimate_translation(mesh, R, K, masks, t_init=None, diameter=None, iters=DEFAULT_ITERS, znear=0.05,
                         return_stats=False, occluders=None):
    """Fit the translation of every rotation hypothesis to its frame's mask (DESIGN.md section 18):
      mesh   a CUDA `nope_b200.vsd.Mesh` (mm, model frame),
      R      [F, P, 3, 3] (or [F, 3, 3] for P = 1), float32 or float64, model -> OpenCV camera,
      K      [F, 3, 3] or [F, 4] (fx, fy, cx, cy), read on the host,
      masks  [F, H, W] uint8 or bool, nonzero = object; (H, W) is the frame size,
      t_init [F, 3] or [F, P, 3] (mm); None: `initial_translation(masks, K, diameter)`,
      iters  updates (default 4), znear as `render_depth`,
      occluders  None, or [F, H, W] uint8 or bool with the masks' shape: nonzero where something may be in front of
             the object (DESIGN.md section 24).  Those pixels count for neither the silhouette nor the mask, so a
             mask cut by an occluder does not pull the fit; None (or all zero) is the plain fit, bit for bit.
    -> (t float64 [F, P, 3], iou float64 [F, P]): the translation after `iters` updates and the silhouette IoU there
    (0 for an empty silhouette); NaN for both where the frame's mask is empty.  With return_stats, also int32
    [F, P, 6]: n_S, |S n M| and the silhouette's box (row0, row1, col0, col1) at the returned t.  With occluders, S and
    M are restricted to the pixels outside them throughout.  Runs on the mesh's device and current stream without
    synchronising."""
    dev = cuda_device(mesh, "estimate_translation")
    R, t_init, k, F_, P, iters = fit_args(mesh, R, t_init, K, iters, znear, t_name="t_init")
    m = _masks(masks)
    if m.shape[0] != F_:
        raise ValueError(f"masks for {F_} frames expected, got {tuple(m.shape)}")
    o = occluder_masks(occluders, m)
    H, W = m.shape[1:]
    if t_init is None and diameter is None:
        raise ValueError("estimate_translation needs t_init or the object diameter")
    with torch.cuda.device(dev):
        m = _to_dev(m, dev, torch.uint8)
        o = None if o is None else _to_dev(o, dev, torch.uint8)
        t0 = broadcast_t(initial_translation(m, k, diameter) if t_init is None else t_init, F_, P, dev)
        Rd = _to_dev(R, dev, torch.float64)
        depth = workspace(dev, F_, P, H, W)
        t = torch.empty((F_, P, 3), device=dev, dtype=torch.float64)
        iou = torch.empty((F_, P), device=dev, dtype=torch.float64)
        stats = torch.empty((F_, P, 6), device=dev, dtype=torch.int32) if return_stats else None
        _lib.check(_lib.load().nope_fit_translation_occluded(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
            _lib.ptr(t0), _lib.ptr(m), _lib.ptr(o), k.data_ptr(), F_, P, H, W, float(znear), iters, _lib.ptr(depth),
            _lib.ptr(t), _lib.ptr(iou), _lib.ptr(stats), _lib.stream(dev)))
    return (t, iou, stats) if return_stats else (t, iou)
