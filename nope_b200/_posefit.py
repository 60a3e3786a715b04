"""The front end the pose fits share: the translation fit, the depth refinement and the contour refinement (DESIGN.md
sections 18-20).  Argument parsing, the geometric tolerance schedule, and the workspace and outputs of one call."""
import math

import numpy as np
import torch

from . import _lib
from .bop import _host_k, _to_dev
from .vsd import MAX_SIDE, Mesh

MAX_BATCH = 65535            # F and P
MAX_ITERS = 1024             # the refinements' bound on iters


def _tensor(x):
    return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)


def _masks(masks):
    m = _tensor(masks)
    if m.dim() == 2:
        m = m[None]
    if m.dim() != 3 or m.shape[0] < 1:
        raise ValueError(f"masks [F, H, W] expected, got {tuple(m.shape)}")
    if m.dtype not in (torch.uint8, torch.bool):
        raise ValueError(f"masks must be uint8 or bool, got {m.dtype}")
    H, W = m.shape[1:]
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"H and W must be in [1, {MAX_SIDE}], got {(H, W)}")
    return m


def cuda_device(mesh, name):
    """the mesh's device, which must be a CUDA device: the fits have no CPU fallback"""
    if not isinstance(mesh, Mesh):
        raise ValueError("mesh must be a nope_b200.vsd.Mesh")
    if mesh.device.type != "cuda":
        raise _lib.NopeError(f"{name} needs a CUDA mesh (no CPU fallback)")
    return mesh.device


def check_iters(iters, max_iters=math.inf):
    if isinstance(iters, bool) or int(iters) != iters or not 0 <= iters <= max_iters:
        raise ValueError(f"iters must be an integer in [0, {max_iters}], got {iters!r}")
    return int(iters)


def fit_args(mesh, R, t, K, iters, znear, max_iters=math.inf, t_name="t"):
    """The arguments every fit takes, checked: a `Mesh`; R [F, P, 3, 3] (or [F, 3, 3] for P = 1), float32 or float64;
    t [F, 3] (shared by the frame's hypotheses), [F, P, 3] or None; iters an integer in [0, max_iters]; znear finite and
    > 0; K as `bop._host_k` takes it.  -> (R [F, P, 3, 3], t, K float64 [F, 4] on the host, F, P, iters)"""
    if not isinstance(mesh, Mesh):
        raise ValueError("mesh must be a nope_b200.vsd.Mesh")
    R = _tensor(R)
    if R.dim() == 3:
        R = R[:, None]
    if R.dim() != 4 or R.shape[2:] != (3, 3) or R.shape[0] < 1 or R.shape[1] < 1:
        raise ValueError(f"R [F, P, 3, 3] or [F, 3, 3] expected, got {tuple(R.shape)}")
    if R.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"R must be float32 or float64, got {R.dtype}")
    F, P = R.shape[:2]
    if F > MAX_BATCH or P > MAX_BATCH:
        raise ValueError(f"F and P must be <= {MAX_BATCH}, got {(F, P)}")
    if t is not None:
        t = _tensor(t)
        if t.shape not in ((F, 3), (F, P, 3)):
            raise ValueError(f"{t_name} [{F}, 3] or [{F}, {P}, 3] expected, got {tuple(t.shape)}")
    iters = check_iters(iters, max_iters)
    if not (np.isfinite(znear) and znear > 0):
        raise ValueError(f"znear must be finite and > 0, got {znear}")
    return R, t, _host_k(K, F), F, P, iters


def broadcast_t(t, F, P, dev):
    """t [F, 3] or [F, P, 3] -> contiguous float64 [F, P, 3] on dev"""
    t = _to_dev(t, dev, torch.float64)
    return t[:, None].expand(F, P, 3).contiguous() if t.dim() == 2 else t


def geometric(end, ratio, iters):
    """end ratio^((iters - i) / max(iters, 1)) for i = 0 ... iters: float64 [iters + 1] from end ratio down to end"""
    i = np.arange(iters + 1, dtype=np.float64)
    return end * ratio ** ((iters - i) / max(iters, 1))


def taus(tau, iters):
    """tau, a number or iters + 1 numbers, all finite and > 0 -> contiguous float64 [iters + 1] on the host"""
    taus = np.asarray(tau.detach().cpu() if torch.is_tensor(tau) else tau, dtype=np.float64).reshape(-1)
    if taus.size == 1:
        taus = np.repeat(taus, iters + 1)
    if taus.size != iters + 1 or not (np.isfinite(taus).all() and (taus > 0).all()):
        raise ValueError(f"tau: one or iters + 1 = {iters + 1} finite numbers > 0 expected, got {taus}")
    return np.ascontiguousarray(taus)


def workspace(dev, F, P, H, W):
    """the rendered depth [F P, H, W] float32 that a fit renders into"""
    return torch.empty((F * P, H, W), device=dev, dtype=torch.float32)


def refine_outputs(dev, F, P, return_sums):
    """R [F, P, 3, 3], t [F, P, 3] and fit [F, P, 4] float64, and the int64 [F, P, 29] sums (None without
    return_sums) of a refinement"""
    f64 = dict(device=dev, dtype=torch.float64)
    sums = torch.empty((F, P, 29), device=dev, dtype=torch.int64) if return_sums else None
    return torch.empty((F, P, 3, 3), **f64), torch.empty((F, P, 3), **f64), torch.empty((F, P, 4), **f64), sums


def pack_refined(R, t, fit, sums, fields):
    out = {name: fit[..., i] for i, name in enumerate(fields)}
    return (R, t, out) if sums is None else (R, t, out, sums)
