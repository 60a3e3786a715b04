"""Pose refinement from the object mask's contour (DESIGN.md section 20), the RGB counterpart of `depth_refine`.  Each
iteration renders every pose hypothesis with the depth rasterizer of `nope_b200.vsd`, pairs each contour pixel of the
rendered silhouette with the frame's object mask through the mask's signed distance field (`mask_sdf`), and takes one
damped Gauss-Newton step of the rotation (about the object's origin) and the translation that moves the contour onto
the mask's.  The pairing tolerance is a fraction of the mask's box size that shrinks from one iteration to the next.
The fit runs on the GPU (`nope_mask_sdf`, `nope_refine_contour_occluded`, csrc/contour_refine.cuh); there is no
CPU fallback."""
import numpy as np
import torch

from . import _lib
from ._posefit import MAX_BATCH, MAX_ITERS, _masks, broadcast_t, check_iters, cuda_device, fit_args, geometric, \
    pack_refined, refine_outputs, taus, workspace
from .translation import occluder_masks
from .bop import _to_dev

DEFAULT_ITERS = 10           # from the convergence table of DESIGN.md section 20
TAU_START = 0.15             # the default schedule: tau_0 = TAU_START s ... tau_iters = TAU_END s, geometric, with
TAU_END = 0.02               # s = sqrt(w h) the mask's box size in px
FIT_FIELDS = ("n_in", "n_contour", "rms", "iou")


def default_tau(iters=DEFAULT_ITERS, start=TAU_START, end=TAU_END):
    """The pairing tolerances float64 [iters + 1], as fractions of the mask's box size: geometric from `start` down to
    `end` (by default TAU_START and TAU_END), so the fit at the returned pose is always scored at `end`."""
    iters = check_iters(iters, MAX_ITERS)
    if not (np.isfinite(start) and np.isfinite(end) and start > 0 and end > 0):
        raise ValueError(f"start and end must be finite and > 0, got {(start, end)}")
    return geometric(end, start / end, iters)


def mask_sdf(masks):
    """The signed distance field float64 [F, H, W] of masks [F, H, W] (or [H, W]; uint8 or bool, nonzero = object) in
    px: sqrt(d2_out) - 1/2 off the object and 1/2 - sqrt(d2_in) on it, where d2_out (d2_in) is the exact squared
    distance to the nearest object (background) pixel of the frame, so the zero level runs along the pixel edges of
    the mask's outline.  NaN everywhere for a mask that is empty or covers the whole frame.  Runs on the masks' device
    (a CUDA device; host masks go to the current one) and current stream without synchronising."""
    m = _masks(masks)
    dev = m.device if m.device.type == "cuda" else None
    if dev is None:
        if not torch.cuda.is_available():
            raise _lib.NopeError("mask_sdf needs a CUDA device (no CPU fallback)")
        dev = torch.device("cuda", torch.cuda.current_device())
    F_, H, W = m.shape
    if F_ > MAX_BATCH:
        raise ValueError(f"F must be <= {MAX_BATCH}, got {F_}")
    with torch.cuda.device(dev):
        md = _to_dev(m, dev, torch.uint8)
        out = torch.empty((F_, H, W), device=dev, dtype=torch.float64)
        _lib.check(_lib.load().nope_mask_sdf(_lib.ptr(md), F_, H, W, _lib.ptr(out), _lib.stream(dev)))
    return out


def refine_pose_contour(mesh, R, t, K, masks, iters=DEFAULT_ITERS, tau=None, znear=0.05, return_sums=False,
                        occluders=None):
    """Refine every pose hypothesis against its frame's object mask (DESIGN.md section 20):
      mesh   a CUDA `nope_b200.vsd.Mesh` (mm, model frame),
      R      [F, P, 3, 3] (or [F, 3, 3] for P = 1), float32 or float64, model -> OpenCV camera,
      t      [F, P, 3] or [F, 3] (shared by the frame's hypotheses), mm,
      K      [F, 3, 3] or [F, 4] (fx, fy, cx, cy), or one for every frame, read on the host,
      masks  [F, H, W] (or [H, W] for F = 1) uint8 or bool, nonzero = object; (H, W) is the frame size,
      iters  updates (default 10); tau: the pairing tolerances as fractions of the mask's box size sqrt(w h), a number
             or iters + 1 numbers (iteration i pairs at tau[i], the returned fit is scored at tau[iters]); None:
             `default_tau(iters)`; znear as `render_depth`,
      occluders  None, or [F, H, W] uint8 or bool with the masks' shape: nonzero where something may be in front of
             the object (DESIGN.md section 24).  The fit then aligns with the mask minus the occluders (its signed
             distance field and box size), and pairs only the contour pixels that, with their four neighbours, lie
             outside them; "n_contour" counts those and "iou" is taken outside them.  None (or all zero) is the plain
             refinement, bit for bit.  `mask_sdf` takes no occluders: pass it the mask minus them.
    -> (R float64 [F, P, 3, 3], t float64 [F, P, 3], fit): the pose after `iters` updates and a dict of float64 [F, P]
    tensors at it: "n_in" the contour pixels paired with the mask, "n_contour" every contour pixel of the render,
    "rms" the RMS distance of the pairs to the mask's outline (px, NaN without pairs) and "iou" the silhouette IoU
    with the mask.  A hypothesis with fewer than 6 pairs keeps its pose; a frame whose mask is empty or full keeps
    every pose, with NaN "rms" and "iou".  With return_sums, also the int64 [F, P, 29] fixed-point sums of the last
    render.  Runs on the mesh's device and current stream without synchronising."""
    R, t, k, F_, P, iters = fit_args(mesh, R, t, K, iters, znear, MAX_ITERS)
    masks = _masks(masks)
    if masks.shape[0] != F_:
        raise ValueError(f"masks [{F_}, H, W] expected, got {tuple(masks.shape)}")
    occ = occluder_masks(occluders, masks)
    H, W = masks.shape[1:]
    tv = taus(default_tau(iters) if tau is None else tau, iters)
    dev = cuda_device(mesh, "refine_pose_contour")
    with torch.cuda.device(dev):
        md = _to_dev(masks, dev, torch.uint8)
        od = None if occ is None else _to_dev(occ, dev, torch.uint8)
        t0 = broadcast_t(t, F_, P, dev)
        Rd = _to_dev(R, dev, torch.float64)
        ws = workspace(dev, F_, P, H, W)
        R_out, t_out, fit, sums = refine_outputs(dev, F_, P, return_sums)
        _lib.check(_lib.load().nope_refine_contour_occluded(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
            _lib.ptr(t0), _lib.ptr(md), _lib.ptr(od), k.data_ptr(), F_, P, H, W, mesh.radius, tv.ctypes.data, iters,
            float(znear), _lib.ptr(ws), _lib.ptr(R_out), _lib.ptr(t_out), _lib.ptr(fit), _lib.ptr(sums),
            _lib.stream(dev)))
    return pack_refined(R_out, t_out, fit, sums, FIT_FIELDS)
