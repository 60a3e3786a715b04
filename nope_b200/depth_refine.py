"""Pose refinement from the sensor depth (DESIGN.md section 19).  Projective point-to-plane ICP of every pose
hypothesis against its frame's depth image: each iteration renders the mesh at the current pose with the depth
rasterizer of `nope_b200.vsd`, pairs each rendered pixel with the sensor reading at the same pixel when the two lie
within a tolerance tau, and takes one damped Gauss-Newton step of the rotation (about the object's origin) and the
translation that minimises the point-to-plane distances of the pairs.  tau shrinks from one iteration to the next.
The fit runs on the GPU (`nope_refine_depth`, csrc/depth_refine.cuh); there is no CPU fallback."""
import numpy as np
import torch

from . import _lib
from ._posefit import MAX_ITERS, _masks, _tensor, broadcast_t, cuda_device, fit_args, geometric, pack_refined, \
    refine_outputs, taus, workspace
from .bop import _to_dev
from .vsd import MAX_SIDE

DEFAULT_ITERS = 6            # from the convergence table of DESIGN.md section 19
TAU_START = 0.5              # the default schedule: tau_0 = TAU_START d ... tau_iters = TAU_END d, geometric
TAU_END = 0.02
FIT_FIELDS = ("n_in", "n_valid", "rms", "score")


def default_tau(diameter, iters=DEFAULT_ITERS):
    """The default pairing tolerances float64 [iters + 1] (mm) for an object of the given diameter (mm): geometric
    from TAU_START d down to TAU_END d, so the fit at the returned pose is always scored at TAU_END d."""
    d = float(diameter)
    if not (np.isfinite(d) and d > 0):
        raise ValueError(f"diameter must be finite and > 0, got {diameter}")
    return geometric(d * TAU_END, TAU_START / TAU_END, iters)


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
    R, t, k, F_, P, iters = fit_args(mesh, R, t, K, iters, znear, MAX_ITERS)
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
    rho = mesh.radius
    tv = taus(default_tau(2.0 * rho, iters) if tau is None else tau, iters)
    dev = cuda_device(mesh, "refine_pose_depth")
    with torch.cuda.device(dev):
        Sd = _to_dev(S, dev, torch.float64)
        md = None if masks is None else _to_dev(masks, dev, torch.uint8)
        t0 = broadcast_t(t, F_, P, dev)
        Rd = _to_dev(R, dev, torch.float64)
        ws = workspace(dev, F_, P, H, W)
        R_out, t_out, fit, sums = refine_outputs(dev, F_, P, return_sums)
        _lib.check(_lib.load().nope_refine_depth(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
            _lib.ptr(t0), _lib.ptr(Sd), _lib.ptr(md), k.data_ptr(), F_, P, H, W, rho, tv.ctypes.data, iters,
            float(znear), _lib.ptr(ws), _lib.ptr(R_out), _lib.ptr(t_out), _lib.ptr(fit), _lib.ptr(sums),
            _lib.stream(dev)))
    return pack_refined(R_out, t_out, fit, sums, FIT_FIELDS)
