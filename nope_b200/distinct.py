"""Distinct pose hypotheses (DESIGN.md section 21): the best-scoring entries of a similarity row such that no two of
their rotations lie within a given angle of each other, modulo the object's symmetry group.  On a pose grid the plain
top-k are nearly always grid neighbours of one mode; these k hypotheses differ, so the stages after the search
(translation, refinement, re-ranking, BOP recall over the top kk) choose among different answers.

Greedy non-maximum suppression in the order of `nope_topk` (descending score, ties -> lowest index): take the best
entry left, drop every entry within theta of it, k times.  Entries scored -inf (not scored, as in the coarse-to-fine
row) or NaN are never taken.  Closeness is the largest trace over the group, compared in float64 against
1 + 2 cos(theta): exact for the continuous axis, not BOP's discretisation of it.  One CUDA kernel
(`nope_distinct_topk`, csrc/distinct.cuh); there is no CPU fallback."""
import math
import numbers

import numpy as np
import torch

from . import _lib
from ._lib import MAX_TOPK
from .bop import _to_dev

MAX_SYM = 32          # discrete rotations per group, the identity included


def symmetry_group(info):
    """(D float64 [n, 3, 3], axis float64 [3]) of one `bop.load_models_info` entry (None: no symmetry): D the
    identity, then the rotation part of each "symmetries_discrete" entry in file order; axis the normalised axis of
    the "symmetries_continuous" entry, zeros without one.  More than one continuous axis is refused."""
    D = [np.eye(3)]
    axis = np.zeros(3)
    if info is not None:
        for m in info.get("symmetries_discrete", []):
            m = np.asarray(m, dtype=np.float64)
            if m.size != 16 or not np.isfinite(m).all():
                raise ValueError("a discrete symmetry must be 16 finite numbers (a 4 x 4 transform)")
            D.append(m.reshape(4, 4)[:3, :3])
        cont = info.get("symmetries_continuous", [])
        if len(cont) > 1:
            raise ValueError(f"at most one continuous symmetry axis is supported, got {len(cont)}")
        if cont:
            a = np.asarray(cont[0]["axis"], dtype=np.float64).reshape(-1)
            if a.shape != (3,) or not np.isfinite(a).all() or not np.linalg.norm(a) > 0:
                raise ValueError("a continuous symmetry axis must be a finite, non-zero 3-vector")
            axis = a / np.linalg.norm(a)
    if len(D) > MAX_SYM:
        raise ValueError(f"at most {MAX_SYM - 1} discrete symmetries are supported, got {len(D) - 1}")
    return np.stack(D), axis


def threshold(min_angle_deg):
    """c_thr = 1 + 2 cos(theta) in float64 for theta = min_angle_deg in [0, 180]"""
    if isinstance(min_angle_deg, bool) or not isinstance(min_angle_deg, numbers.Real) or \
            not 0.0 <= float(min_angle_deg) <= 180.0:
        raise ValueError(f"min_angle_deg must be a number in [0, 180], got {min_angle_deg!r}")
    return 1.0 + 2.0 * math.cos(math.radians(float(min_angle_deg)))


def distinct_topk(sim, rotations, k, min_angle_deg, symmetries=None):
    """Distinct top-k of every row of sim [..., N] (float32, CUDA):
      sim        [B, N], [B, Q, N] or [Q, N] (the query forms of `predict_pose`); for the in-plane search the caller
                 flattens [..., A, N] to [..., A * N];
      rotations  [B | 1, N, 3, 3] object -> camera rotations of the entries; rotations[b] serves every row of sim[b]
                 (row block b of sim's first dimension), rotations[0] every row when the first dimension is 1;
      k          1 .. 64;  min_angle_deg: theta in [0, 180] degrees;
      symmetries None (no symmetry), one `bop.load_models_info` entry for every row, or a list of one entry per
                 index of sim's first dimension.
    -> (score float32 [..., k], idx int64 [..., k]) in sim's leading shape, padded with (-inf, -1) when fewer than k
    distinct entries are scored.  Runs on sim's device and current stream without synchronising."""
    if not torch.is_tensor(sim) or sim.dim() < 1 or sim.dim() > 3 or sim.shape[-1] < 1:
        raise ValueError(f"sim [N], [B, N] or [B, Q, N] (a torch tensor) expected, got "
                         f"{tuple(sim.shape) if torch.is_tensor(sim) else type(sim).__name__}")
    if sim.dtype != torch.float32:
        raise ValueError(f"sim must be float32, got {sim.dtype}")
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= MAX_TOPK:
        raise ValueError(f"k must be an integer in [1, {MAX_TOPK}], got {k!r}")
    c_thr = threshold(min_angle_deg)
    lead, N = tuple(sim.shape[:-1]), sim.shape[-1]
    R = math.prod(lead)
    B = lead[0] if lead else 1
    if R < 1:
        raise ValueError(f"sim has no rows: {tuple(sim.shape)}")
    rot = torch.as_tensor(np.asarray(rotations) if not torch.is_tensor(rotations) else rotations)
    if rot.dim() != 4 or rot.shape[1:] != (N, 3, 3) or rot.shape[0] not in (1, B):
        raise ValueError(f"rotations [{B} or 1, {N}, 3, 3] expected, got {tuple(rot.shape)}")
    G_r = rot.shape[0]
    if symmetries is None or isinstance(symmetries, dict):
        groups, group = [symmetry_group(symmetries)], np.zeros(R, dtype=np.int32)
    else:
        symmetries = list(symmetries)
        if len(symmetries) != B:
            raise ValueError(f"symmetries: None, one models_info entry or a list of {B} expected, got a list of "
                             f"{len(symmetries)}")
        groups = [symmetry_group(s) for s in symmetries]
        group = np.repeat(np.arange(B, dtype=np.int32), R // B)
    disc = np.ascontiguousarray(np.concatenate([g[0] for g in groups]), dtype=np.float64)
    n_disc = np.array([len(g[0]) for g in groups], dtype=np.int32)
    axis = np.ascontiguousarray(np.stack([g[1] for g in groups]), dtype=np.float64)
    if sim.device.type != "cuda":
        raise _lib.NopeError("distinct_topk needs a CUDA similarity (no CPU fallback)")
    dev = sim.device
    with torch.cuda.device(dev):
        s = sim.contiguous()
        rd = _to_dev(rot, dev, torch.float64)
        score = torch.empty(lead + (k,), device=dev, dtype=torch.float32)
        idx = torch.empty(lead + (k,), device=dev, dtype=torch.int64)
        _lib.check(_lib.load().nope_distinct_topk(
            _lib.ptr(s), R, N, _lib.ptr(rd), G_r, R // G_r, disc.ctypes.data, n_disc.ctypes.data, axis.ctypes.data,
            len(groups), group.ctypes.data, k, c_thr, _lib.ptr(idx), _lib.ptr(score), _lib.stream(dev)))
    return score, idx
