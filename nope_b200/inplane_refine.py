"""Joint roll and viewpoint refinement (DESIGN.md section 14).

The in-plane search (section 11) returns poses Rz(alpha_a) * template_poses[n]: its error cannot fall below the
angle bins combined with the grid spacing.  This search continues from each (reference, query) row's best (angle,
pose) pairs.  The viewpoint is refined on the template side, with a 3x3 lattice of small rotations about the camera's
x and y axes (no roll is ever asked of the UNet); the roll is refined on the query side, by encoding the query crop
rotated by the centre's roll +- a shrinking step.

A candidate is (D, seed, rho): D an accumulated rotation, seed a grid index, rho = (cos, sin) a roll.  Its relative
rotation is D * S_seed (as in section 10), its query latent the encoding of the crop rotated by rho (the section 11
image convention), and the pose it stands for R = Rz(rho) * D * template_poses[seed].  Each step scores every
(angle slot, pose slot) pair of one multi-query sweep and keeps the best distinct pairs.  The centre pair (identity
pose slot, unchanged roll) is swept with the same pose bits and the same latent bits as before, so a row's best score
never decreases and never falls below its best in-plane search score.
"""
import itertools
import math
import numbers

import numpy as np
import torch

from . import _lib
from ._lib import MAX_TOPK
from .inplane import check_angles, inplane_table
from .refine import axis_angle_matrix, grid_constants, identity_centres
from .search import query_rows, row_pairs

XY = 9              # pose slots per centre: the 3x3 xy lattice, identity first, then lexicographic (i, j)
ROLL = 3            # angle slots per centre: rho, rho + phi, rho - phi
MAX_KEEP = 16
_XY_OFFSETS = [(0, 0)] + [v for v in itertools.product((-1, 0, 1), repeat=2) if v != (0, 0)]


def xy_stencil(theta):
    """[9, 3, 3] float64: exp([theta * (i, j, 0)]x) for i, j in {-1, 0, 1}, the identity first."""
    return np.stack([axis_angle_matrix(theta * np.array([i, j, 0.0])) for i, j in _XY_OFFSETS])


class InplaneRefiner:
    """The per-step constants of a joint roll and viewpoint refinement over one pose grid and A angle bins.

    Step s uses the viewpoint lattice spacing theta_s = theta0 * 2^-s (theta0 as in PoseRefiner: half the grid's
    median nearest-neighbour angle) and its xy stencil (float32 [9, 9]); the roll step phi_s = (pi / A) 2^-s (half a
    bin at s = 0) as float32 (cos, sin); and the trace threshold fp32(1 + 2 cos(psi_s / 2)), psi_s = min(theta_s,
    phi_s), above which two candidates count as one.  All computed once on the host in float64; device copies are
    made on first use."""

    def __init__(self, template_poses, angles=36, steps=4):
        self.angles = check_angles(angles)
        if isinstance(steps, bool) or not isinstance(steps, numbers.Integral) or steps < 1:
            raise ValueError(f"steps must be a positive integer, got {steps!r}")
        self.steps = int(steps)
        self.template_poses, self.theta0, self.thetas = grid_constants(template_poses, self.steps)
        self.num_poses = int(self.template_poses.shape[0])
        self.phi0 = math.pi / self.angles
        self.phis = tuple(self.phi0 * 2.0 ** -s for s in range(self.steps))
        self.stencils = torch.from_numpy(np.stack([xy_stencil(t).reshape(XY, 9) for t in self.thetas])
                                         .astype(np.float32))
        self.rolls = tuple((float(np.float32(math.cos(p))), float(np.float32(math.sin(p)))) for p in self.phis)
        self.thresholds = tuple(float(np.float32(1.0 + 2.0 * math.cos(min(t, p) / 2.0)))
                                for t, p in zip(self.thetas, self.phis))
        self._device = {}

    def hypotheses(self, keep):
        """UNet hypotheses (templates) one row sweeps in the refinement steps: keep * 9 per step"""
        return self.steps * keep * XY

    def crops(self, keep):
        """query crops one row encodes in the refinement steps: 2 * keep per step"""
        return self.steps * keep * (ROLL - 1)

    def _on(self, device):
        key = str(device)
        if key not in self._device:
            self._device[key] = (self.stencils.to(device), self.template_poses.to(device),
                                 inplane_table(self.angles).to(device))
        return self._device[key]


def check_inplane_refine_args(refiner, all_relativeR, keep, k, B=None):
    """ValueError for arguments a refinement cannot run with (checked on the host, before any device work)."""
    if not isinstance(refiner, InplaneRefiner):
        raise ValueError("refiner must be a nope_b200.inplane_refine.InplaneRefiner")
    n = refiner.num_poses
    if all_relativeR.dim() != 3 or all_relativeR.shape[1] != n or all_relativeR.shape[2] != 6:
        raise ValueError(f"all_relativeR must be [B, {n}, 6] (the refiner's grid), got {tuple(all_relativeR.shape)}")
    if B is not None and all_relativeR.shape[0] != B:
        raise ValueError(f"all_relativeR has {all_relativeR.shape[0]} references, the reference batch {B}")
    for name, v, hi in (("keep", keep, MAX_KEEP), ("k", k, MAX_TOPK)):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not 1 <= v <= hi:
            raise ValueError(f"{name} must be an integer in [1, {hi}], got {v!r}")
    if keep > refiner.angles * n:
        raise ValueError(f"keep ({keep}) exceeds the {refiner.angles} x {n} (angle, pose) pairs")
    if k > XY * ROLL * keep * keep:
        raise ValueError(f"k ({k}) exceeds the {XY * ROLL * keep * keep} pairs of keep = {keep}")



def rotate_pairs(images, image_idx, cossin):
    """images [B, 3, H, W] (CUDA), image_idx [P] (int), cossin [P, 2] (float32) -> [P, 3, H, W] float32: image
    image_idx[p] rotated by cossin[p] (inplane_rotate_pairs_kernel, materialised; the refinement itself never forms
    these crops), all -1 for an index outside [0, B)."""
    if images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"images [B, 3, H, W] expected, got {tuple(images.shape)}")
    if image_idx.dim() != 1 or tuple(cossin.shape) != (image_idx.shape[0], 2) or image_idx.shape[0] < 1:
        raise ValueError(f"image_idx [P] and cossin [P, 2] expected, got {tuple(image_idx.shape)} and "
                         f"{tuple(cossin.shape)}")
    if images.device.type != "cuda":
        raise _lib.NopeError("rotate_pairs needs CUDA tensors (no CPU fallback)")
    dev = images.device
    x = images.to(torch.float32).contiguous()
    idx = image_idx.to(dev, torch.int32).contiguous()
    cs = cossin.to(dev, torch.float32).contiguous()
    B, _, H, W = x.shape
    out = torch.empty((idx.shape[0], 3, H, W), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_inplane_rotate_pairs(_lib.ptr(x), B, H, W, _lib.ptr(idx), _lib.ptr(cs),
                                                         idx.shape[0], _lib.ptr(out), _lib.stream(dev)))
    return out


def propose(D, seed, cossin, all_relativeR, stencil_, roll, Q):
    """nope_pose_refine_inplane_propose: centres D [R, keep, 9] float32 / seed [R, keep] int32 / cossin [R, keep, 2],
    all_relativeR [B, N, 6], stencil_ [9, 9], roll = (cos, sin) of the step -> dict(D [R, keep * 9, 9], seed,
    rel [R, keep * 9, 9], poses [R, keep * 9, 6], cossin [R, keep * 3, 2])."""
    R, keep = seed.shape
    B, N = all_relativeR.shape[0], all_relativeR.shape[1]
    P = keep * XY
    dev = all_relativeR.device
    out = {"D": torch.empty((R, P, 9), device=dev, dtype=torch.float32),
           "seed": torch.empty((R, P), device=dev, dtype=torch.int32),
           "rel": torch.empty((R, P, 9), device=dev, dtype=torch.float32),
           "poses": torch.empty((R, P, 6), device=dev, dtype=torch.float32),
           "cossin": torch.empty((R, keep * ROLL, 2), device=dev, dtype=torch.float32)}
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_refine_inplane_propose(
            _lib.ptr(D), _lib.ptr(seed), _lib.ptr(cossin), R, keep, _lib.ptr(all_relativeR), B, Q, N,
            _lib.ptr(stencil_), float(roll[0]), float(roll[1]), _lib.ptr(out["D"]), _lib.ptr(out["seed"]),
            _lib.ptr(out["rel"]), _lib.ptr(out["poses"]), _lib.ptr(out["cossin"]), _lib.stream(dev)))
    return out


def select(sim, cand, threshold, k):
    """nope_pose_refine_inplane_select: sim [R, keep * 3, keep * 9] scored at the pairs of propose() -> dict(D [R, k,
    9], seed [R, k] int32, cossin [R, k, 2], aslot [R, k] int32, score [R, k], rel [R, k, 9]); -inf / -1 / zeros past
    the last distinct pair."""
    R, A3, P = sim.shape
    keep = P // XY
    dev = sim.device
    out = {"D": torch.empty((R, k, 9), device=dev, dtype=torch.float32),
           "seed": torch.empty((R, k), device=dev, dtype=torch.int32),
           "cossin": torch.empty((R, k, 2), device=dev, dtype=torch.float32),
           "aslot": torch.empty((R, k), device=dev, dtype=torch.int32),
           "score": torch.empty((R, k), device=dev, dtype=torch.float32),
           "rel": torch.empty((R, k, 9), device=dev, dtype=torch.float32)}
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_pose_refine_inplane_select(
            _lib.ptr(sim), _lib.ptr(cand["D"]), _lib.ptr(cand["seed"]), _lib.ptr(cand["rel"]),
            _lib.ptr(cand["cossin"]), R, keep, k, float(threshold), _lib.ptr(out["D"]), _lib.ptr(out["seed"]),
            _lib.ptr(out["cossin"]), _lib.ptr(out["aslot"]), _lib.ptr(out["score"]), _lib.ptr(out["rel"]),
            _lib.stream(dev)))
    return out


def check_centres(seeds, lead):
    """ValueError unless seeds is refine_inplane's dict of explicit centres for rows of shape `lead` (checked on the
    host): D float32 [*lead, keep, 3, 3], seed integer [*lead, keep], cossin float32 [*lead, keep, 2].  -> keep"""
    if set(seeds) != {"D", "seed", "cossin"} or not all(torch.is_tensor(v) for v in seeds.values()):
        raise ValueError(f"centre seeds must be a dict of tensors D, seed and cossin, got keys {sorted(seeds)}")
    D, seed, cs = seeds["D"], seeds["seed"], seeds["cossin"]
    if seed.is_floating_point() or seed.is_complex() or seed.dtype == torch.bool:
        raise ValueError(f"seeds['seed'] must be an integer tensor, got {seed.dtype}")
    if D.dtype != torch.float32 or cs.dtype != torch.float32:
        raise ValueError(f"seeds['D'] and seeds['cossin'] must be float32, got {D.dtype} and {cs.dtype}")
    keep = int(seed.shape[-1]) if seed.dim() == len(lead) + 1 else 0
    if keep < 1 or tuple(seed.shape) != lead + (keep,) or tuple(D.shape) != lead + (keep, 3, 3) or \
            tuple(cs.shape) != lead + (keep, 2):
        raise ValueError(f"centre seeds D {lead + ('keep', 3, 3)}, seed {lead + ('keep',)} and cossin "
                         f"{lead + ('keep', 2)} expected, got {tuple(D.shape)}, {tuple(seed.shape)} and "
                         f"{tuple(cs.shape)}")
    return keep


def _check_seed_latents(seed_latents, shape):
    if tuple(seed_latents.shape) != shape:
        raise ValueError(f"seed_latents must be {shape}, got {tuple(seed_latents.shape)}")


def refine_inplane(engine, encoder, ref_feat, query_images, all_relativeR, seeds, seed_latents, refiner, k=5,
                   hidden=None):
    """Refine each (reference, query) row from its best (angle, pose) pairs, with any engine that has `sweep()`.

    ref_feat [B, C, 32, 32]; query_images [B, 3, 256, 256] or [B, Q, 3, 256, 256]; all_relativeR [B, N, 6], the grid
    of `refiner`; seeds = (pose_idx, angle_idx), each [B(, Q), keep] (keep = their last dimension, e.g. the joint
    top-keep of the in-plane search), or explicit centres dict(D [B(, Q), keep, 3, 3] float32, seed [B(, Q), keep]
    integer, cossin [B(, Q), keep, 2] float32), e.g. track.seed_centres of prior rotations ((pose_idx, angle_idx) is
    the centre (I, pose_idx, inplane_table(A)[angle_idx])); seed_latents [B(, Q), keep, C, 32, 32], the latents of
    the crops rotated by the seeds' rolls (for the tuple, the search's latents of those angle copies, gathered, not
    re-encoded); encoder: a FeatureExtractor on the native engine.
    -> dict(D [B(, Q), k, 3, 3], seed [B(, Q), k] int64, cossin [B(, Q), k, 2], score [B(, Q), k], rel6d [B(, Q), k,
    6] and latent [B(, Q), k, C, 32, 32] (the pose and query latent each score was swept at), hypotheses and crops
    (per row, by the steps)).  Descending score; ranks past the last distinct pair have score -inf and seed -1.

    Each step proposes keep * 9 poses and keep * 3 rolls per row, encodes the 2 * keep new rolled crops, sweeps all
    pairs with one reference row per (reference, query) and selects the next `keep` centres (the last step: k).
    Everything runs on the current stream with no host synchronisation (device copies of the refiner's constants
    are made by the first call on a device).  hidden [B(, Q), 256, 256] (uint8 or bool, the crops' masks of pixels
    that may be hidden, DESIGN.md section 27): every step's pairs score over the visible map of their own roll, made
    from the candidates' (cos, sin) by latent_visibility, so a kept roll and a fresh one use the same arithmetic."""
    centres = isinstance(seeds, dict)
    rest = tuple(ref_feat.shape[1:])
    if centres:
        lead = query_rows(query_images, ref_feat, (3, 256, 256))[1]
        keep = check_centres(seeds, lead)
        _check_seed_latents(seed_latents, lead + (keep,) + rest)
    else:
        pose_idx, angle_idx = seeds
        keep = int(pose_idx.shape[-1])
    check_inplane_refine_args(refiner, all_relativeR, keep, k, ref_feat.shape[0])
    dev = engine.device
    _, _, Q, lead, ref_rows, images = row_pairs(dev, ref_feat, query_images, (3, 256, 256))
    if not centres and (tuple(pose_idx.shape) != lead + (keep,) or tuple(angle_idx.shape) != lead + (keep,)):
        raise ValueError(f"seeds must be two {lead + (keep,)} tensors, got {tuple(pose_idx.shape)} and "
                         f"{tuple(angle_idx.shape)}")
    _check_seed_latents(seed_latents, lead + (keep,) + rest)
    if hidden is not None:
        from .visibility import check_hidden, latent_visibility
        hid = check_hidden(hidden, lead, "refine_inplane").to(dev)
    rows = ref_rows.shape[0]
    stencils, _, table = refiner._on(dev)
    rel = all_relativeR.to(dev, torch.float32).contiguous()
    if centres:
        cur = {"D": seeds["D"].to(dev).reshape(rows, keep, 9).contiguous(),
               "seed": seeds["seed"].to(dev).reshape(rows, keep).to(torch.int32),
               "cossin": seeds["cossin"].to(dev).reshape(rows, keep, 2).contiguous()}
    else:
        cur = {"D": identity_centres(rows, keep, dev),
               "seed": pose_idx.to(dev).reshape(rows, keep).to(torch.int32),
               "cossin": table[angle_idx.to(dev).reshape(rows, keep)].contiguous()}
    lat = seed_latents.to(dev, torch.float32).reshape(rows, keep, *rest)
    row_ix = torch.arange(rows, device=dev)
    for s in range(refiner.steps):
        n = int(cur["seed"].shape[1])
        cand = propose(cur["D"], cur["seed"], cur["cossin"], rel, stencils[s], refiner.rolls[s], Q)
        fresh_cs = cand["cossin"].view(rows, n, ROLL, 2)[:, :, 1:].reshape(rows * n * (ROLL - 1), 2)
        fresh_idx = row_ix.to(torch.int32)[:, None].expand(rows, n * (ROLL - 1)).reshape(-1)
        fresh = encoder.encode_image_rotated(images, fresh_idx, fresh_cs).view(rows, n, ROLL - 1, *rest)
        qf = torch.cat([lat[:, :, None], fresh], dim=2).view(rows, n * ROLL, *rest)
        vis = {}                                   # query_visible= only with a mask: any sweep() serves without one
        if hidden is not None:
            pair_idx = row_ix.to(torch.int32)[:, None].expand(rows, n * ROLL).reshape(-1)
            vis["query_visible"] = latent_visibility(hid, cand["cossin"].reshape(-1, 2), pair_idx).view(
                rows, n * ROLL, 32, 32)
        sim = engine.sweep(ref_rows, cand["poses"], query_feat=qf, want_emb=False, want_sim=True, k=0, **vis)["sim"]
        cur = select(sim, cand, refiner.thresholds[s], k if s == refiner.steps - 1 else keep)
        lat = qf[row_ix[:, None], cur["aslot"].long().clamp_min(0)]
    return {"D": cur["D"].view(*lead, k, 3, 3), "seed": cur["seed"].to(torch.int64).view(*lead, k),
            "cossin": cur["cossin"].view(*lead, k, 2), "score": cur["score"].view(*lead, k),
            "rel6d": cur["rel"][..., :6].reshape(*lead, k, 6), "latent": lat.view(*lead, k, *rest),
            "hypotheses": refiner.hypotheses(keep), "crops": refiner.crops(keep)}


def pose_rotations(D, seed, cossin, refiner):
    """R = Rz(rho) * D * template_poses[seed] [..., 3, 3] in float64 (zeros where seed is -1), with Rz(rho) =
    [[c, -s, 0], [s, c, 0], [0, 0, 1]] of the float32 (c, s)."""
    _, tp, _ = refiner._on(D.device)
    cs = cossin.to(torch.float64)
    c, s = cs[..., 0], cs[..., 1]
    Rz = torch.zeros(cs.shape[:-1] + (3, 3), device=D.device, dtype=torch.float64)
    Rz[..., 0, 0], Rz[..., 0, 1], Rz[..., 1, 0], Rz[..., 1, 1], Rz[..., 2, 2] = c, -s, s, c, 1.0
    return Rz @ D.to(torch.float64) @ tp[seed.clamp_min(0)]


def roll_degrees(cossin):
    """atan2(sin, cos) in degrees, float64"""
    cs = cossin.to(torch.float64)
    return torch.rad2deg(torch.atan2(cs[..., 1], cs[..., 0]))
