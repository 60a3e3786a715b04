"""BOP 2019 average recall (DESIGN.md section 15): the object symmetries of a dataset's `models_info.json`, the
symmetry-aware MSSD / MSPD errors on the GPU (pose_error.cuh) and the recall averages of the BOP 2019 protocol
(Hodan et al.), AR = (AR_VSD + AR_MSSD + AR_MSPD) / 3.  The definitions follow the protocol as published; agreement
with the BOP toolkit's code is not verified (DESIGN.md section 15 lists where it might differ)."""
import json
import math

import numpy as np
import torch

from . import _lib

# the recall thresholds: float64 values of numpy.arange, so ties at exactly a threshold depend on their last bits
VSD_TAUS = np.arange(0.05, 0.51, 0.05)          # x diameter: the misalignment tolerances of AR_VSD
VSD_THETAS = np.arange(0.05, 0.51, 0.05)        # VSD correctness thresholds
MSSD_THETAS = np.arange(0.05, 0.51, 0.05)       # x diameter
MSPD_THETAS = np.arange(5, 51, 5).astype(np.float64)   # x W / 640 px
MAX_SYM_DISC_STEP = 0.01


def load_models_info(path):
    """A BOP `models_info.json` -> {obj_id (int): {"diameter": float (mm), "symmetries_discrete": [4 x 4 float64
    arrays], "symmetries_continuous": [{"axis": float64 [3], "offset": float64 [3]}]}}.  Missing symmetry keys mean
    none; every other key of an entry is dropped."""
    with open(path) as fh:
        raw = json.load(fh)
    if not isinstance(raw, dict):
        raise ValueError(f"{path}: a JSON object keyed by object id expected")
    out = {}
    for key, entry in raw.items():
        try:
            obj_id = int(key)
        except ValueError:
            raise ValueError(f"{path}: object id {key!r} is not an integer") from None
        if "diameter" not in entry:
            raise ValueError(f"{path}: object {obj_id} has no diameter")
        diameter = float(entry["diameter"])
        if not (math.isfinite(diameter) and diameter > 0):
            raise ValueError(f"{path}: object {obj_id} has diameter {diameter}, a finite value > 0 expected")
        disc = []
        for m in entry.get("symmetries_discrete", []):
            m = np.asarray(m, dtype=np.float64)
            if m.size != 16 or not np.isfinite(m).all():
                raise ValueError(f"{path}: object {obj_id}: a discrete symmetry must be 16 finite numbers")
            disc.append(m.reshape(4, 4))
        cont = []
        for c in entry.get("symmetries_continuous", []):
            axis = np.asarray(c["axis"], dtype=np.float64).reshape(-1)
            offset = np.asarray(c.get("offset", [0.0, 0.0, 0.0]), dtype=np.float64).reshape(-1)
            if axis.shape != (3,) or offset.shape != (3,) or not (np.isfinite(axis).all() and np.isfinite(offset).all()):
                raise ValueError(f"{path}: object {obj_id}: a continuous symmetry needs a finite 3-vector axis and offset")
            if not np.linalg.norm(axis) > 0:
                raise ValueError(f"{path}: object {obj_id}: a continuous symmetry axis must be non-zero")
            cont.append({"axis": axis, "offset": offset})
        out[obj_id] = {"diameter": diameter, "symmetries_discrete": disc, "symmetries_continuous": cont}
    return out


def _rodrigues(axis, angle):
    a = axis / np.linalg.norm(axis)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + math.sin(angle) * k + (1.0 - math.cos(angle)) * (k @ k)


def symmetry_transformations(info, max_sym_disc_step=MAX_SYM_DISC_STEP):
    """float64 [S, 3, 4] (R | t, model frame, mm) of one entry of `load_models_info`.
    Discrete set: the identity, then every `symmetries_discrete` entry in file order.  Continuous set: for each
    `symmetries_continuous` entry in file order, n = ceil(pi / max_sym_disc_step) rotations about the normalised axis
    at angles i * 2 pi / n, i = 0 ... n - 1 (Rodrigues), with t = offset - R offset; angle 0 is included.  The result
    is transform c * D + d = (R_c R_d, R_c t_d + t_c) for continuous c and discrete d; without a continuous symmetry,
    the discrete set."""
    if not max_sym_disc_step > 0:
        raise ValueError(f"max_sym_disc_step must be > 0, got {max_sym_disc_step}")
    disc = [(np.eye(3), np.zeros(3))] + [(m[:3, :3].copy(), m[:3, 3].copy()) for m in info.get("symmetries_discrete", [])]
    cont = []
    n = int(math.ceil(math.pi / max_sym_disc_step))
    for c in info.get("symmetries_continuous", []):
        offset = np.asarray(c["offset"], dtype=np.float64)
        for i in range(n):
            R = _rodrigues(np.asarray(c["axis"], dtype=np.float64), i * 2.0 * math.pi / n)
            cont.append((R, offset - R @ offset))
    if not cont:
        cont = [(np.eye(3), np.zeros(3))]
    out = np.empty((len(cont) * len(disc), 3, 4))
    for ci, (Rc, tc) in enumerate(cont):
        for di, (Rd, td) in enumerate(disc):
            out[ci * len(disc) + di, :, :3] = Rc @ Rd
            out[ci * len(disc) + di, :, 3] = Rc @ td + tc
    return out


def _host_k(K, F):
    """-> contiguous float64 [F, 4] (fx, fy, cx, cy) on the host, checked"""
    k = torch.as_tensor(np.asarray(K) if not torch.is_tensor(K) else K).detach().cpu().to(torch.float64)
    if k.shape in ((3, 3), (4,)):
        k = k[None]
    if k.dim() == 3 and k.shape[1:] == (3, 3):
        k = torch.stack([k[:, 0, 0], k[:, 1, 1], k[:, 0, 2], k[:, 1, 2]], dim=1)
    if k.dim() != 2 or k.shape[1] != 4:
        raise ValueError(f"K [F, 3, 3], [3, 3], [F, 4] or [4] expected, got {tuple(k.shape)}")
    if k.shape[0] == 1 and F > 1:
        k = k.expand(F, 4)
    if k.shape[0] != F:
        raise ValueError(f"K for {F} rows expected, got {tuple(k.shape)}")
    k = k.contiguous()
    if not torch.isfinite(k).all() or (k[:, :2] == 0).any():
        raise ValueError("intrinsics must be finite with fx and fy non-zero")
    return k


def _to_dev(x, dev, dtype):
    x = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
    if x.device.type == "cpu" and dev.type == "cuda":
        return x.to(dtype).contiguous().pin_memory().to(dev, non_blocking=True)
    return x.to(device=dev, dtype=dtype).contiguous()


def pose_errors(points, R_est, t_est, R_gt, t_gt, K, syms):
    """Symmetry-aware MSSD (mm) and MSPD (px), float64 [F, P] each, of P estimated poses per row:
      points [V, 3] (model points, mm; a CUDA tensor, e.g. `Mesh.vertices`, or host data; used as float32),
      R_est [F, P, 3, 3], t_est [F, P, 3] or [F, 3] (shared by the row's estimates) or [F, 3, 1],
      R_gt [F, 3, 3], t_gt [F, 3] or [F, 3, 1]   (model -> OpenCV camera),
      K [F, 3, 3], [F, 4] (fx, fy, cx, cy), or one of them for every row, read on the host,
      syms [S, 3, 4] (`symmetry_transformations`).
    MSSD = min_s max_x |(R_e x + t_e) - (R_g (R_s x + t_s) + t_g)|, MSPD the same between projections; an MSPD is
    +inf when a point lies at Z <= 0 under every symmetry of the ground truth or under the estimate.  Runs on the
    points' device (or the current CUDA device), on the current stream, without synchronising."""
    pts = torch.as_tensor(np.asarray(points) if not torch.is_tensor(points) else points)
    if pts.dim() != 2 or pts.shape[1] != 3 or pts.shape[0] < 1:
        raise ValueError(f"points [V, 3] with V >= 1 expected, got {tuple(pts.shape)}")
    R_est = torch.as_tensor(np.asarray(R_est) if not torch.is_tensor(R_est) else R_est)
    R_gt = torch.as_tensor(np.asarray(R_gt) if not torch.is_tensor(R_gt) else R_gt)
    t_est = torch.as_tensor(np.asarray(t_est) if not torch.is_tensor(t_est) else t_est)
    t_gt = torch.as_tensor(np.asarray(t_gt) if not torch.is_tensor(t_gt) else t_gt)
    if R_est.dim() != 4 or R_est.shape[2:] != (3, 3) or R_est.shape[0] < 1 or R_est.shape[1] < 1:
        raise ValueError(f"R_est [F, P, 3, 3] expected, got {tuple(R_est.shape)}")
    F_, P = R_est.shape[:2]
    if F_ > 65535 or P > 65535:
        raise ValueError(f"F and P must be <= 65535, got {(F_, P)}")
    if R_gt.shape != (F_, 3, 3):
        raise ValueError(f"R_gt [{F_}, 3, 3] expected, got {tuple(R_gt.shape)}")
    if t_gt.shape == (F_, 3, 1):
        t_gt = t_gt[..., 0]
    if t_gt.shape != (F_, 3):
        raise ValueError(f"t_gt [{F_}, 3] or [{F_}, 3, 1] expected, got {tuple(t_gt.shape)}")
    if t_est.shape == (F_, 3, 1):
        t_est = t_est[..., 0]
    if t_est.shape == (F_, 3):
        t_est = t_est[:, None].expand(F_, P, 3)
    if t_est.shape != (F_, P, 3):
        raise ValueError(f"t_est [{F_}, {P}, 3], [{F_}, 3] or [{F_}, 3, 1] expected, got {tuple(t_est.shape)}")
    sy = torch.as_tensor(np.asarray(syms) if not torch.is_tensor(syms) else syms)
    if sy.dim() != 3 or sy.shape[1:] != (3, 4) or not 1 <= sy.shape[0] <= 1 << 24:
        raise ValueError(f"syms [S, 3, 4] with 1 <= S <= 2^24 expected, got {tuple(sy.shape)}")
    k = _host_k(K, F_)
    dev = pts.device if pts.device.type == "cuda" else (
        R_est.device if R_est.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device()))
    if dev.type != "cuda":
        raise _lib.NopeError("pose_errors runs on a CUDA device (no CPU fallback)")
    with torch.cuda.device(dev):
        p = _to_dev(pts, dev, torch.float32)
        gt = torch.cat([_to_dev(R_gt, dev, torch.float64), _to_dev(t_gt, dev, torch.float64)[..., None]], dim=2)
        est = torch.cat([_to_dev(R_est, dev, torch.float64), _to_dev(t_est, dev, torch.float64)[..., None]], dim=3)
        gt, est = gt.contiguous(), est.contiguous()
        s = _to_dev(sy, dev, torch.float64)
        mssd = torch.empty((F_, P), device=dev, dtype=torch.float64)
        mspd = torch.empty((F_, P), device=dev, dtype=torch.float64)
        _lib.check(_lib.load().nope_pose_errors(
            _lib.ptr(p), p.shape[0], _lib.ptr(s), s.shape[0], _lib.ptr(gt), _lib.ptr(est), k.data_ptr(), F_, P,
            _lib.ptr(mssd), _lib.ptr(mspd), _lib.stream(dev)))
    return mssd, mspd


def _np(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def average_recall(vsd, mssd, mspd, diameter, width):
    """BOP 2019 average recalls (fractions in [0, 1]) of B targets, each with k estimates scored by the per-metric
    minimum over its k estimates (k = 1: the BOP figure):
      vsd [B, k, 10] (VSD at tau = VSD_TAUS x diameter), mssd [B, k] (mm), mspd [B, k] (px),
      diameter: float or [B] (mm), width: image width W (px).
    An error e is correct when e < theta (strict).  -> {"ar_vsd", "ar_mssd", "ar_mspd", "ar"}."""
    vsd, mssd, mspd = _np(vsd).astype(np.float64), _np(mssd).astype(np.float64), _np(mspd).astype(np.float64)
    if vsd.ndim != 3 or vsd.shape[2] != len(VSD_TAUS) or mssd.shape != vsd.shape[:2] or mspd.shape != vsd.shape[:2]:
        raise ValueError(f"vsd [B, k, {len(VSD_TAUS)}], mssd [B, k] and mspd [B, k] expected, got {vsd.shape}, "
                         f"{mssd.shape}, {mspd.shape}")
    B = vsd.shape[0]
    if B < 1 or vsd.shape[1] < 1:
        raise ValueError("empty batch")
    diam = np.broadcast_to(np.asarray(diameter, dtype=np.float64), (B,))
    if not (np.isfinite(diam).all() and (diam > 0).all()):
        raise ValueError("diameter must be finite and > 0")
    if not float(width) > 0:
        raise ValueError(f"width must be > 0, got {width}")
    e_vsd, e_mssd, e_mspd = vsd.min(1), mssd.min(1), mspd.min(1)                 # [B, 10], [B], [B]
    ar_vsd = float(np.mean(e_vsd[:, :, None] < VSD_THETAS[None, None, :]))       # 100 (tau, theta) recalls
    ar_mssd = float(np.mean(e_mssd[:, None] < MSSD_THETAS[None, :] * diam[:, None]))
    ar_mspd = float(np.mean(e_mspd[:, None] < MSPD_THETAS[None, :] * (float(width) / 640.0)))
    return {"ar_vsd": ar_vsd, "ar_mssd": ar_mssd, "ar_mspd": ar_mspd, "ar": (ar_vsd + ar_mssd + ar_mspd) / 3.0}
