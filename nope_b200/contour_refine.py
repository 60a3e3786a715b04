"""Pose refinement from the object mask's contour (DESIGN.md section 20), the RGB counterpart of `depth_refine`.  Each
iteration renders every pose hypothesis with the depth rasterizer of `nope_b200.vsd`, pairs each contour pixel of the
rendered silhouette with the frame's object mask through the mask's signed distance field (`mask_sdf`), and takes one
damped Gauss-Newton step of the rotation (about the object's origin) and the translation that moves the contour onto
the mask's.  The pairing tolerance is a fraction of the mask's box size that shrinks from one iteration to the next.
The fit runs on the GPU (`nope_mask_sdf`, `nope_refine_contour`, csrc/contour_refine.cuh); there is no CPU
fallback."""
import numpy as np
import torch

from . import _lib
from .bop import _host_k, _to_dev
from .depth_refine import MAX_ITERS, _tensor
from .translation import MAX_BATCH, _masks
from .vsd import Mesh, _stream

DEFAULT_ITERS = 10           # from the convergence table of DESIGN.md section 20
TAU_START = 0.15             # the default schedule: tau_0 = TAU_START s ... tau_iters = TAU_END s, geometric, with
TAU_END = 0.02               # s = sqrt(w h) the mask's box size in px
FIT_FIELDS = ("n_in", "n_contour", "rms", "iou")


def default_tau(iters=DEFAULT_ITERS, start=TAU_START, end=TAU_END):
    """The pairing tolerances float64 [iters + 1], as fractions of the mask's box size: geometric from `start` down to
    `end` (by default TAU_START and TAU_END), so the fit at the returned pose is always scored at `end`."""
    if isinstance(iters, bool) or int(iters) != iters or not 0 <= iters <= MAX_ITERS:
        raise ValueError(f"iters must be an integer in [0, {MAX_ITERS}], got {iters!r}")
    if not (np.isfinite(start) and np.isfinite(end) and start > 0 and end > 0):
        raise ValueError(f"start and end must be finite and > 0, got {(start, end)}")
    iters = int(iters)
    i = np.arange(iters + 1, dtype=np.float64)
    return end * (start / end) ** ((iters - i) / max(iters, 1))


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
        _lib.check(_lib.load().nope_mask_sdf(_lib.ptr(md), F_, H, W, _lib.ptr(out), _stream(dev)))
    return out


def refine_pose_contour(mesh, R, t, K, masks, iters=DEFAULT_ITERS, tau=None, znear=0.05, return_sums=False):
    """Refine every pose hypothesis against its frame's object mask (DESIGN.md section 20):
      mesh   a CUDA `nope_b200.vsd.Mesh` (mm, model frame),
      R      [F, P, 3, 3] (or [F, 3, 3] for P = 1), float32 or float64, model -> OpenCV camera,
      t      [F, P, 3] or [F, 3] (shared by the frame's hypotheses), mm,
      K      [F, 3, 3] or [F, 4] (fx, fy, cx, cy), or one for every frame, read on the host,
      masks  [F, H, W] (or [H, W] for F = 1) uint8 or bool, nonzero = object; (H, W) is the frame size,
      iters  updates (default 10); tau: the pairing tolerances as fractions of the mask's box size sqrt(w h), a number
             or iters + 1 numbers (iteration i pairs at tau[i], the returned fit is scored at tau[iters]); None:
             `default_tau(iters)`; znear as `render_depth`.
    -> (R float64 [F, P, 3, 3], t float64 [F, P, 3], fit): the pose after `iters` updates and a dict of float64 [F, P]
    tensors at it: "n_in" the contour pixels paired with the mask, "n_contour" every contour pixel of the render,
    "rms" the RMS distance of the pairs to the mask's outline (px, NaN without pairs) and "iou" the silhouette IoU
    with the mask.  A hypothesis with fewer than 6 pairs keeps its pose; a frame whose mask is empty or full keeps
    every pose, with NaN "rms" and "iou".  With return_sums, also the int64 [F, P, 29] fixed-point sums of the last
    render.  Runs on the mesh's device and current stream without synchronising."""
    if not isinstance(mesh, Mesh):
        raise ValueError("mesh must be a nope_b200.vsd.Mesh")
    R = _tensor(R)
    if R.dim() == 3:
        R = R[:, None]
    if R.dim() != 4 or R.shape[2:] != (3, 3) or R.shape[0] < 1 or R.shape[1] < 1:
        raise ValueError(f"R [F, P, 3, 3] or [F, 3, 3] expected, got {tuple(R.shape)}")
    if R.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"R must be float32 or float64, got {R.dtype}")
    F_, P = R.shape[:2]
    if F_ > MAX_BATCH or P > MAX_BATCH:
        raise ValueError(f"F and P must be <= {MAX_BATCH}, got {(F_, P)}")
    t = _tensor(t)
    if t.shape not in ((F_, 3), (F_, P, 3)):
        raise ValueError(f"t [{F_}, 3] or [{F_}, {P}, 3] expected, got {tuple(t.shape)}")
    masks = _masks(masks)
    if masks.shape[0] != F_:
        raise ValueError(f"masks [{F_}, H, W] expected, got {tuple(masks.shape)}")
    H, W = masks.shape[1:]
    if isinstance(iters, bool) or int(iters) != iters or not 0 <= iters <= MAX_ITERS:
        raise ValueError(f"iters must be an integer in [0, {MAX_ITERS}], got {iters!r}")
    iters = int(iters)
    if not (np.isfinite(znear) and znear > 0):
        raise ValueError(f"znear must be finite and > 0, got {znear}")
    k = _host_k(K, F_)
    taus = default_tau(iters) if tau is None else np.asarray(
        tau.detach().cpu() if torch.is_tensor(tau) else tau, dtype=np.float64).reshape(-1)
    if taus.size == 1:
        taus = np.repeat(taus, iters + 1)
    if taus.size != iters + 1 or not (np.isfinite(taus).all() and (taus > 0).all()):
        raise ValueError(f"tau: one or iters + 1 = {iters + 1} finite numbers > 0 expected, got {taus}")
    taus = np.ascontiguousarray(taus)
    dev = mesh.device
    if dev.type != "cuda":
        raise _lib.NopeError("refine_pose_contour needs a CUDA mesh (no CPU fallback)")
    with torch.cuda.device(dev):
        md = _to_dev(masks, dev, torch.uint8)
        t0 = _to_dev(t, dev, torch.float64)
        t0 = t0[:, None].expand(F_, P, 3).contiguous() if t0.dim() == 2 else t0
        Rd = _to_dev(R, dev, torch.float64)
        ws = torch.empty((F_ * P, H, W), device=dev, dtype=torch.float32)
        R_out = torch.empty((F_, P, 3, 3), device=dev, dtype=torch.float64)
        t_out = torch.empty((F_, P, 3), device=dev, dtype=torch.float64)
        fit = torch.empty((F_, P, 4), device=dev, dtype=torch.float64)
        sums = torch.empty((F_, P, 29), device=dev, dtype=torch.int64) if return_sums else None
        _lib.check(_lib.load().nope_refine_contour(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
            _lib.ptr(t0), _lib.ptr(md), k.data_ptr(), F_, P, H, W, mesh.radius, taus.ctypes.data, iters,
            float(znear), _lib.ptr(ws), _lib.ptr(R_out), _lib.ptr(t_out), _lib.ptr(fit), _lib.ptr(sums),
            _stream(dev)))
    out = {name: fit[..., i] for i, name in enumerate(FIT_FIELDS)}
    return (R_out, t_out, out, sums) if return_sums else (R_out, t_out, out)
