"""Off-grid pose refinement (DESIGN.md section 10).

A grid search can only return grid poses: its error is bounded below by the grid spacing.  The score of the UNet is
continuous in the pose, so the search can continue between grid poses.  Each (reference, query) row starts from its
best `keep` grid poses; each step scores a 3x3x3 lattice of small rotations around every kept pose, keeps the best
`keep` distinct ones, and halves the lattice spacing.

A candidate is (D, seed): `seed` a grid index, D an accumulated rotation.  Its relative rotation is D * S_seed
(S_seed the seed's relative rotation) and its template pose D * template_poses[seed].  The centre of every lattice
is re-proposed with the identity and re-scored to the same bits, so a row's best score never decreases from one
step to the next.  A hypothesis's score does not depend on the other hypotheses of its launch, so every refined pose
has exactly the score a separate sweep of it gives.
"""
import itertools

import numpy as np
import torch

from . import _lib
from ._lib import MAX_TOPK
from .hierarchy import rotation_trace
from .search import row_pairs

STENCIL = 27        # the 3x3x3 lattice: slot 0 the identity, then the other 26 in lexicographic (i, j, l) order
_OFFSETS = [(0, 0, 0)] + [v for v in itertools.product((-1, 0, 1), repeat=3) if v != (0, 0, 0)]


def nearest_neighbour_angles(R):
    """Geodesic angle (radians, float64) from each rotation of R [N, 3, 3] to its nearest other rotation."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 9)
    best = []
    for i in range(0, len(R), 256):                # 256 rows at a time bound the [rows, N, 9] products
        t = rotation_trace(R[i:i + 256], R)
        t[np.arange(t.shape[0]), np.arange(i, i + t.shape[0])] = -np.inf
        best.append(t.max(axis=1))
    return np.arccos(np.clip((np.concatenate(best) - 1.0) / 2.0, -1.0, 1.0))


def axis_angle_matrix(w):
    """exp([w]x) for w [3] (radians), float64, by Rodrigues' formula; exactly I for w = 0."""
    w = np.asarray(w, dtype=np.float64)
    phi = float(np.linalg.norm(w))
    if phi == 0.0:
        return np.eye(3)
    x, y, z = w / phi
    K = np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])
    return np.eye(3) + np.sin(phi) * K + (1.0 - np.cos(phi)) * (K @ K)


def stencil(theta):
    """[27, 3, 3] float64: exp([theta * (i, j, l)]x) for i, j, l in {-1, 0, 1}, the identity first."""
    return np.stack([axis_angle_matrix(theta * np.asarray(v, dtype=np.float64)) for v in _OFFSETS])


def grid_constants(template_poses, steps):
    """The grid constants of a refiner over template_poses [N >= 2, 3, 3] with `steps` (checked) steps: ->
    (template_poses float64 on the host, theta0 = half the grid's median nearest-neighbour geodesic angle, thetas =
    theta0 * 2^-s for each step s)."""
    R = np.asarray(template_poses.cpu().numpy() if torch.is_tensor(template_poses) else template_poses,
                   dtype=np.float64)
    if R.ndim != 3 or R.shape[1:] != (3, 3) or R.shape[0] < 2:
        raise ValueError(f"template_poses must be [N >= 2, 3, 3], got {tuple(R.shape)}")
    theta0 = 0.5 * float(np.median(nearest_neighbour_angles(R)))
    return torch.from_numpy(R.copy()), theta0, tuple(theta0 * 2.0 ** -s for s in range(steps))


def identity_centres(rows, keep, device):
    """The first step's centres D: the identity for each of a row's `keep` seeds, float32 [rows, keep, 9]"""
    return torch.eye(3, device=device, dtype=torch.float32).reshape(1, 1, 9).expand(rows, keep, 9).contiguous()


class PoseRefiner:
    """The per-step constants of a refinement over one pose grid.

    template_poses [N, 3, 3]: the grid's template rotations.  theta0 is half the grid's median nearest-neighbour
    geodesic angle; step s uses the lattice spacing theta0 * 2^-s, its stencil (float32 [27, 9]) and the trace
    threshold fp32(1 + 2 cos(theta_s / 2)) above which two candidates count as one (closer than theta_s / 2).
    All computed once on the host in float64; device copies are made on first use."""

    def __init__(self, template_poses, steps=4):
        if int(steps) != steps or steps < 1:
            raise ValueError(f"steps must be a positive integer, got {steps}")
        self.steps = int(steps)
        self.template_poses, self.theta0, self.thetas = grid_constants(template_poses, self.steps)
        self.num_poses = int(self.template_poses.shape[0])
        self.stencils = torch.from_numpy(np.stack([stencil(t).reshape(STENCIL, 9) for t in self.thetas])
                                         .astype(np.float32))
        self.thresholds = tuple(float(np.float32(1.0 + 2.0 * np.cos(t / 2.0))) for t in self.thetas)
        self._device = {}

    def hypotheses(self, keep):
        """Hypotheses one (reference, query) row sweeps: the seed grid, then keep * 27 per step."""
        return self.num_poses + self.steps * keep * STENCIL

    def _on(self, device):
        key = str(device)
        if key not in self._device:
            self._device[key] = (self.stencils.to(device), self.template_poses.to(device))
        return self._device[key]


def check_refine_args(refiner, all_relativeR, keep, k, B=None):
    """ValueError for arguments a refinement cannot run with (checked on the host, before any device work)."""
    if not isinstance(refiner, PoseRefiner):
        raise ValueError("refiner must be a nope_b200.refine.PoseRefiner")
    n = refiner.num_poses
    if all_relativeR.dim() != 3 or all_relativeR.shape[1] != n or all_relativeR.shape[2] != 6:
        raise ValueError(f"all_relativeR must be [B, {n}, 6] (the refiner's grid), got {tuple(all_relativeR.shape)}")
    if B is not None and all_relativeR.shape[0] != B:
        raise ValueError(f"all_relativeR has {all_relativeR.shape[0]} references, the reference batch {B}")
    if not 1 <= keep <= MAX_TOPK:
        raise ValueError(f"keep must be in [1, {MAX_TOPK}], got {keep}")
    if keep > n:
        raise ValueError(f"keep ({keep}) exceeds the grid ({n} poses)")
    if not 1 <= k <= MAX_TOPK:
        raise ValueError(f"k must be in [1, {MAX_TOPK}], got {k}")
    if k > keep * STENCIL:
        raise ValueError(f"k ({k}) exceeds the {keep * STENCIL} candidates of keep = {keep}")


def propose(D, seed, all_relativeR, stencil_, Q):
    """nope_pose_refine_propose: centres D [R, keep, 9] float32 / seed [R, keep] int32, all_relativeR [B, N, 6],
    stencil_ [27, 9] -> dict(D [R, M, 9], seed [R, M] int32, rel [R, M, 9], poses [R, M, 6]), M = keep * 27."""
    R, keep = seed.shape
    B, N = all_relativeR.shape[0], all_relativeR.shape[1]
    M = keep * STENCIL
    dev = all_relativeR.device
    out = {"D": torch.empty((R, M, 9), device=dev, dtype=torch.float32),
           "seed": torch.empty((R, M), device=dev, dtype=torch.int32),
           "rel": torch.empty((R, M, 9), device=dev, dtype=torch.float32),
           "poses": torch.empty((R, M, 6), device=dev, dtype=torch.float32)}
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_refine_propose(
            _lib.ptr(D), _lib.ptr(seed), R, keep, _lib.ptr(all_relativeR), B, Q, N, _lib.ptr(stencil_),
            _lib.ptr(out["D"]), _lib.ptr(out["seed"]), _lib.ptr(out["rel"]), _lib.ptr(out["poses"]),
            _lib.stream(dev)))
    return out


def select(sim, cand, threshold, k):
    """nope_pose_refine_select: sim [R, M] scored at the candidates of propose() -> dict(D [R, k, 9],
    seed [R, k] int32, score [R, k], rel [R, k, 9]); -inf / -1 / zeros past the last distinct candidate."""
    R, M = sim.shape
    dev = sim.device
    out = {"D": torch.empty((R, k, 9), device=dev, dtype=torch.float32),
           "seed": torch.empty((R, k), device=dev, dtype=torch.int32),
           "score": torch.empty((R, k), device=dev, dtype=torch.float32),
           "rel": torch.empty((R, k, 9), device=dev, dtype=torch.float32)}
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_refine_select(
            _lib.ptr(sim), _lib.ptr(cand["D"]), _lib.ptr(cand["seed"]), _lib.ptr(cand["rel"]), R, M, k,
            float(threshold), _lib.ptr(out["D"]), _lib.ptr(out["seed"]), _lib.ptr(out["score"]), _lib.ptr(out["rel"]),
            _lib.stream(dev)))
    return out


def refine(engine, ref_feat, query_feat, all_relativeR, seed_idx, refiner, k=5):
    """Refine each (reference, query) row from its seeds, with any engine that has `sweep()` (UNet, UNetModelPose).

    ref_feat [B, C, 32, 32]; query_feat [B, C, 32, 32] or [B, Q, C, 32, 32]; all_relativeR [B, N, 6], the grid of
    `refiner`; seed_idx [B(, Q), keep] grid indices (keep = its last dimension, e.g. the top-keep of a sweep).
    -> dict(D [B(, Q), k, 3, 3], seed [B(, Q), k] int64, score [B(, Q), k], rel6d [B(, Q), k, 6] (the pose each
    score was swept at), hypotheses: swept per row by the refinement steps).  Descending score; ranks past the
    last distinct candidate have score -inf, seed -1 and D = 0.

    Each step proposes keep * 27 candidates per row, sweeps them with one reference row per (reference, query)
    (Q = 1) and selects the next `keep` centres (the last step: k).  Everything runs on the current stream with no
    host synchronisation (device copies of the refiner's constants are made by the first call on a device)."""
    keep = int(seed_idx.shape[-1])
    check_refine_args(refiner, all_relativeR, keep, k, ref_feat.shape[0])
    dev = engine.device
    _, _, Q, lead, ref_rows, query_rows_ = row_pairs(dev, ref_feat, query_feat)
    if tuple(seed_idx.shape[:-1]) != lead:
        raise ValueError(f"seed_idx must be {lead + (keep,)} for these queries, got {tuple(seed_idx.shape)}")
    rows = ref_rows.shape[0]
    rel = all_relativeR.to(dev, torch.float32).contiguous()
    stencils, _ = refiner._on(dev)
    cur = {"D": identity_centres(rows, keep, dev), "seed": seed_idx.to(dev).reshape(rows, keep).to(torch.int32)}
    for s in range(refiner.steps):
        cand = propose(cur["D"], cur["seed"], rel, stencils[s], Q)
        sim = engine.sweep(ref_rows, cand["poses"], query_feat=query_rows_, want_emb=False, want_sim=True,
                           k=0)["sim"]
        cur = select(sim, cand, refiner.thresholds[s], k if s == refiner.steps - 1 else keep)
    return {"D": cur["D"].view(*lead, k, 3, 3), "seed": cur["seed"].to(torch.int64).view(*lead, k),
            "score": cur["score"].view(*lead, k), "rel6d": cur["rel"][..., :6].reshape(*lead, k, 6),
            "hypotheses": refiner.steps * keep * STENCIL}


def template_rotations(D, seed, refiner):
    """R = D * template_poses[seed] [..., 3, 3] in float64 (zeros where seed is -1)."""
    _, tp = refiner._on(D.device)
    return D.to(torch.float64) @ tp[seed.clamp_min(0)]
