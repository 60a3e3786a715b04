"""Coarse-to-fine pose search over nested pose grids (DESIGN.md section 9).

The exhaustive sweep pays for every pose of the grid.  With a hierarchy of grids (the reference ships
icospheres of 42 / 162 / 642 / 2562 poses, nested), a search scores the coarsest grid, keeps its best `keep`
poses per (reference, query) row, and sweeps only the finer poses around them, level by level.

Every fine pose is assigned to its nearest coarse pose (its *cell*); cells are disjoint, so the union of a row's
`keep` cells needs no deduplication.  A pose's score does not depend on the other hypotheses of its launch, so each
pose the search scores gets exactly the score the exhaustive sweep gives it: the search differs from the exhaustive
one only in which poses it scores.
"""

import numpy as np
import torch

from . import _lib
from ._lib import MAX_TOPK
from .search import row_pairs


def rotation_trace(fine_R, coarse_R):
    """trace(R_f R_c^T) [N_fine, N_coarse] in float64, the nine products summed left to right.  The geodesic angle
    arccos((trace - 1) / 2) decreases as it grows.  Icosphere grids hold exact ties (a fine pose midway between
    two coarse ones), so the summation order is fixed: a matrix product would break those ties by its own order."""
    f = np.asarray(fine_R, dtype=np.float64).reshape(-1, 1, 9)
    c = np.asarray(coarse_R, dtype=np.float64).reshape(1, -1, 9)
    p = f * c
    t = p[..., 0].copy()
    for j in range(1, 9):
        t += p[..., j]
    return t


def cell_table(coarse_R, fine_R):
    """int32 [N_coarse, F]: row i lists (ascending, -1 padded) the fine poses whose nearest coarse pose is i, by
    SO(3) geodesic angle (the largest rotation_trace); ties go to the lowest coarse index.  Float64 on the host.
    F is the largest cell."""
    c = np.asarray(coarse_R, dtype=np.float64).reshape(-1, 9)
    f = np.asarray(fine_R, dtype=np.float64).reshape(-1, 9)
    # argmax takes the first (lowest) index of a tie; 256 fine poses at a time bound the [rows, N_coarse, 9] products
    nearest = np.concatenate([np.argmax(rotation_trace(f[i:i + 256], c), axis=1) for i in range(0, len(f), 256)])
    order = np.argsort(nearest, kind="stable")         # fine indices ascending inside each cell
    counts = np.bincount(nearest, minlength=c.shape[0])
    F = int(counts.max())
    table = np.full((c.shape[0], F), -1, dtype=np.int32)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    for i in range(c.shape[0]):
        table[i, :counts[i]] = order[starts[i]:starts[i] + counts[i]]
    return table


class PoseHierarchy:
    """Cell tables between consecutive levels of a pose-grid hierarchy.

    levels: two or more rotation sets [N_l, 3, 3] (template rotations), coarsest first.  Relative rotations
    R_t R_ref^-1 keep geodesic distances, so the tables built from the template rotations serve every reference
    of a batch.  Device copies are made on first use."""

    def __init__(self, levels):
        levels = [np.asarray(R.cpu().numpy() if torch.is_tensor(R) else R, dtype=np.float64) for R in levels]
        if len(levels) < 2:
            raise ValueError(f"a pose hierarchy needs at least two levels, got {len(levels)}")
        for l, R in enumerate(levels):
            if R.ndim != 3 or R.shape[1:] != (3, 3) or R.shape[0] < 1:
                raise ValueError(f"level {l}: rotations [N, 3, 3] expected, got {tuple(R.shape)}")
        self.sizes = tuple(int(R.shape[0]) for R in levels)
        self._tables = [cell_table(levels[l], levels[l + 1]) for l in range(len(levels) - 1)]
        self._device = {}

    @property
    def num_levels(self):
        return len(self.sizes)

    def cell_width(self, step):
        """F of the step from level `step` to `step + 1`: the largest cell."""
        return int(self._tables[step].shape[1])

    def cells(self, step):
        """The cell table of the step from level `step` to `step + 1` (a copy; int32 [N_step, F], -1 padded)."""
        return torch.from_numpy(self._tables[step].copy())

    def hypotheses(self, keep):
        """Hypotheses one (reference, query) row sweeps: the whole coarsest grid, then keep * F per finer level."""
        return self.sizes[0] + sum(keep * self.cell_width(s) for s in range(self.num_levels - 1))

    def _cells_on(self, step, device):
        key = (step, str(device))
        if key not in self._device:
            self._device[key] = torch.from_numpy(self._tables[step]).to(device)
        return self._device[key]


def check_search_args(hierarchy, all_relativeR_levels, keep, k):
    """ValueError for arguments a search cannot run with (checked on the host, before any device work)."""
    if not isinstance(hierarchy, PoseHierarchy):
        raise ValueError("hierarchy must be a nope_b200.hierarchy.PoseHierarchy")
    if len(all_relativeR_levels) < 2:
        raise ValueError(f"a coarse-to-fine search needs at least two levels, got {len(all_relativeR_levels)}")
    if len(all_relativeR_levels) != hierarchy.num_levels:
        raise ValueError(f"{len(all_relativeR_levels)} pose levels for a hierarchy of {hierarchy.num_levels}")
    for l, (p, n) in enumerate(zip(all_relativeR_levels, hierarchy.sizes)):
        if p.dim() != 3 or p.shape[1] != n or p.shape[2] != 6:
            raise ValueError(f"all_relativeR_levels[{l}] must be [B, {n}, 6], got {tuple(p.shape)}")
    if not 1 <= keep <= MAX_TOPK:
        raise ValueError(f"keep must be in [1, {MAX_TOPK}], got {keep}")
    if keep > hierarchy.sizes[0]:
        raise ValueError(f"keep ({keep}) exceeds the coarsest grid ({hierarchy.sizes[0]} poses)")
    if not 1 <= k <= MAX_TOPK:
        raise ValueError(f"k must be in [1, {MAX_TOPK}], got {k}")


def expand(top_idx, cells, poses, Q, M):
    """nope_pose_cells_expand: top_idx [R, keep] int64, cells [N_coarse, F] int32, poses [B, n_fine, 6] ->
    (cand [R, M] int32, poses [R, M, 6])."""
    R, keep = top_idx.shape
    B, n_fine = poses.shape[0], poses.shape[1]
    dev = poses.device
    cand = torch.empty((R, M), device=dev, dtype=torch.int32)
    out = torch.empty((R, M, 6), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_cells_expand(
            _lib.ptr(top_idx), R, keep, _lib.ptr(cells), cells.shape[0], cells.shape[1], _lib.ptr(poses), B, Q,
            n_fine, M, _lib.ptr(cand), _lib.ptr(out), _lib.stream(dev)))
    return cand, out


def rank(sim, cand, n_fine, k, want_sim=True):
    """nope_pose_cells_rank: sim [R, M] at fine indices cand [R, M] -> (sim over the fine grid [R, n_fine] with
    -inf where nothing was scored | None, topv [R, k], topi [R, k] int64)."""
    R, M = sim.shape
    dev = sim.device
    out_sim = torch.empty((R, n_fine), device=dev, dtype=torch.float32) if want_sim else None
    topv = torch.empty((R, k), device=dev, dtype=torch.float32)
    topi = torch.empty((R, k), device=dev, dtype=torch.int64)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_cells_rank(
            _lib.ptr(sim), _lib.ptr(cand), R, M, n_fine, k, _lib.ptr(out_sim), _lib.ptr(topv), _lib.ptr(topi),
            _lib.stream(dev)))
    return out_sim, topv, topi


def search(engine, ref_feat, query_feat, all_relativeR_levels, hierarchy, keep=8, k=5):
    """Coarse-to-fine search with any engine that has `sweep()` (UNet, UNetModelPose).

    ref_feat [B, C, 32, 32]; query_feat [B, C, 32, 32] or [B, Q, C, 32, 32]; all_relativeR_levels[l] [B, N_l, 6].
    -> dict(sim [B(, Q), N_L] with -inf at poses that were not scored, topv / topi [B(, Q), k] as indices of the
    finest grid, ties -> lowest index, hypotheses: swept per (reference, query) row).

    Stage 0 sweeps the coarsest grid and keeps each row's top `keep`; stage l >= 1 sweeps the union of their
    cells at level l (keep * F_l slots per row, one reference per row with its query) and ranks it.  Everything
    runs on the current stream; all sizes are known on the host, so nothing waits for the device."""
    check_search_args(hierarchy, all_relativeR_levels, keep, k)
    B = ref_feat.shape[0]
    for l, p in enumerate(all_relativeR_levels):
        if p.shape[0] != B:
            raise ValueError(f"all_relativeR_levels[{l}] has {p.shape[0]} references, ref_feat {B}")
    dev = engine.device
    ref_feat, query_feat, Q, lead, ref_rows, query_rows_ = row_pairs(dev, ref_feat, query_feat)
    levels = [p.to(dev, torch.float32).contiguous() for p in all_relativeR_levels]
    top = engine.sweep(ref_feat, levels[0], query_feat=query_feat, want_emb=False, want_sim=False,
                       k=keep)["topi"].reshape(B * Q, keep)
    last = hierarchy.num_levels - 1
    sim = topv = None
    for l in range(1, last + 1):
        cells = hierarchy._cells_on(l - 1, dev)
        M = keep * cells.shape[1]
        cand, poses = expand(top, cells, levels[l], Q, M)
        scored = engine.sweep(ref_rows, poses, query_feat=query_rows_, want_emb=False, want_sim=True, k=0)["sim"]
        sim, topv, top = rank(scored, cand, hierarchy.sizes[l], k if l == last else keep, want_sim=l == last)
    n = hierarchy.sizes[-1]
    return {"sim": sim.view(*lead, n), "topv": topv.view(*lead, k), "topi": top.view(*lead, k),
            "hypotheses": hierarchy.hypotheses(keep)}
