"""Pose refinement from the sensor depth (DESIGN.md section 19).  Projective point-to-plane ICP of every pose
hypothesis against its frame's depth image: each iteration renders the mesh at the current pose with the depth
rasterizer of `nope_b200.vsd`, pairs each rendered pixel with the sensor reading at the same pixel when the two lie
within a tolerance tau, and takes one damped Gauss-Newton step of the rotation (about the object's origin) and the
translation that minimises the point-to-plane distances of the pairs.  tau shrinks from one iteration to the next.
The fit runs on the GPU (`nope_refine_depth`, csrc/depth_refine.cuh); there is no CPU fallback."""
import numpy as np
import torch

from . import _lib
from .bop import _host_k, _to_dev
from .translation import MAX_BATCH, _masks
from .vsd import MAX_SIDE, Mesh, _stream

DEFAULT_ITERS = 6            # from the convergence table of DESIGN.md section 19
TAU_START = 0.5              # the default schedule: tau_0 = TAU_START d ... tau_iters = TAU_END d, geometric
TAU_END = 0.02
MAX_ITERS = 1024
FIT_FIELDS = ("n_in", "n_valid", "rms", "score")


def default_tau(diameter, iters=DEFAULT_ITERS):
    """The default pairing tolerances float64 [iters + 1] (mm) for an object of the given diameter (mm): geometric
    from TAU_START d down to TAU_END d, so the fit at the returned pose is always scored at TAU_END d."""
    d = float(diameter)
    if not (np.isfinite(d) and d > 0):
        raise ValueError(f"diameter must be finite and > 0, got {diameter}")
    i = np.arange(iters + 1, dtype=np.float64)
    return d * TAU_END * (TAU_START / TAU_END) ** ((iters - i) / max(iters, 1))


def _tensor(x):
    return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)


def refine_pose_depth(mesh, R, t, K, depth, masks=None, iters=DEFAULT_ITERS, tau=None, znear=0.05,
                      return_sums=False):
    """Refine every pose hypothesis against its frame's sensor depth (DESIGN.md section 19):
      mesh   a CUDA `nope_b200.vsd.Mesh` (mm, model frame),
      R      [F, P, 3, 3] (or [F, 3, 3] for P = 1), float32 or float64, model -> OpenCV camera,
      t      [F, P, 3] or [F, 3] (shared by the frame's hypotheses), mm,
      K      [F, 3, 3] or [F, 4] (fx, fy, cx, cy), or one for every frame, read on the host,
      depth  [F, H, W] (or [H, W] for F = 1) sensor depth in mm, 0 = no reading (e.g. a BOP depth PNG / 10),
      masks  [F, H, W] uint8 or bool, nonzero = object; None: every pixel counts,
      iters  updates (default 6); tau: the pairing tolerances in mm, a number or iters + 1 numbers (iteration i pairs
             at tau[i], the returned fit is scored at tau[iters]); None: `default_tau(2 rho, iters)` with rho the
             largest vertex norm (`Mesh.radius`); znear as `render_depth`.
    -> (R float64 [F, P, 3, 3], t float64 [F, P, 3], fit): the pose after `iters` updates and a dict of float64 [F, P]
    tensors at it: "n_in" the pairs, "n_valid" the mask pixels with a reading, "rms" the point-to-plane RMS of the
    pairs (mm, NaN without pairs) and "score" = n_in / n_valid (NaN when n_valid = 0).  A hypothesis with fewer than
    6 pairs keeps its pose.  With return_sums, also the int64 [F, P, 29] fixed-point sums of the last render.  Runs on
    the mesh's device and current stream without synchronising."""
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
    S = _tensor(depth)
    if S.dim() == 2:
        S = S[None]
    if S.dim() != 3 or S.shape[0] != F_ or not S.is_floating_point():
        raise ValueError(f"depth: a floating-point [{F_}, H, W] image expected, got {tuple(S.shape)} {S.dtype}")
    H, W = S.shape[1:]
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"H and W must be in [1, {MAX_SIDE}], got {(H, W)}")
    if masks is not None:
        masks = _masks(masks)
        if tuple(masks.shape) != (F_, H, W):
            raise ValueError(f"masks [{F_}, {H}, {W}] expected, got {tuple(masks.shape)}")
    if isinstance(iters, bool) or int(iters) != iters or not 0 <= iters <= MAX_ITERS:
        raise ValueError(f"iters must be an integer in [0, {MAX_ITERS}], got {iters!r}")
    iters = int(iters)
    if not (np.isfinite(znear) and znear > 0):
        raise ValueError(f"znear must be finite and > 0, got {znear}")
    k = _host_k(K, F_)
    rho = mesh.radius
    taus = default_tau(2.0 * rho, iters) if tau is None else np.asarray(
        tau.detach().cpu() if torch.is_tensor(tau) else tau, dtype=np.float64).reshape(-1)
    if taus.size == 1:
        taus = np.repeat(taus, iters + 1)
    if taus.size != iters + 1 or not (np.isfinite(taus).all() and (taus > 0).all()):
        raise ValueError(f"tau: one or iters + 1 = {iters + 1} finite numbers > 0 expected, got {taus}")
    taus = np.ascontiguousarray(taus)
    dev = mesh.device
    if dev.type != "cuda":
        raise _lib.NopeError("refine_pose_depth needs a CUDA mesh (no CPU fallback)")
    with torch.cuda.device(dev):
        Sd = _to_dev(S, dev, torch.float64)
        md = None if masks is None else _to_dev(masks, dev, torch.uint8)
        t0 = _to_dev(t, dev, torch.float64)
        t0 = t0[:, None].expand(F_, P, 3).contiguous() if t0.dim() == 2 else t0
        Rd = _to_dev(R, dev, torch.float64)
        ws = torch.empty((F_ * P, H, W), device=dev, dtype=torch.float32)
        R_out = torch.empty((F_, P, 3, 3), device=dev, dtype=torch.float64)
        t_out = torch.empty((F_, P, 3), device=dev, dtype=torch.float64)
        fit = torch.empty((F_, P, 4), device=dev, dtype=torch.float64)
        sums = torch.empty((F_, P, 29), device=dev, dtype=torch.int64) if return_sums else None
        _lib.check(_lib.load().nope_refine_depth(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
            _lib.ptr(t0), _lib.ptr(Sd), _lib.ptr(md), k.data_ptr(), F_, P, H, W, rho, taus.ctypes.data, iters,
            float(znear), _lib.ptr(ws), _lib.ptr(R_out), _lib.ptr(t_out), _lib.ptr(fit), _lib.ptr(sums),
            _stream(dev)))
    out = {name: fit[..., i] for i, name in enumerate(FIT_FIELDS)}
    return (R_out, t_out, out, sums) if return_sums else (R_out, t_out, out)
