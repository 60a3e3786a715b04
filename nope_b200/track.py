"""Pose tracking (DESIGN.md section 26): refine each frame's roll and viewpoint from the previous frame's poses
instead of searching again.

The joint roll and viewpoint refinement (section 14) only needs centres.  After a search, they come from its
top-`keep` (angle bin, grid pose) pairs; in a video, the previous frame's rotations are already within a few degrees
of the new pose.  `seed_centres` maps each prior rotation to the centre of the section 14 form nearest to it
(track_seed_kernel), `track_inplane` refines from those centres, and `PoseTracker` keeps the previous poses of every
track and searches only the detections it has not seen or has lost.  Per detection, tracking costs keep * (1 + 2 *
steps) encodes and 9 * keep * steps UNet hypotheses, against the A rotated copies a search encodes.
"""
import numbers

import torch

from . import _lib
from .inplane_refine import MAX_KEEP, InplaneRefiner, check_inplane_refine_args, refine_inplane


def seed_centres(R_crop, refiner):
    """The refinement centres of prior rotations R_crop [..., 3, 3] (float32 or float64, CUDA; in the crop camera):
    dict(D [..., 3, 3] float32, seed [...] int32, cossin [..., 2] float32) with Rz(rho) D T[seed] = R_crop up to the
    float32 rounding of D and (cos, sin), T = refiner.template_poses and Rz(rho) = [[c, -s, 0], [s, c, 0], [0, 0, 1]].
    The seed is the grid pose that, at its best roll, lies nearest to the prior, so D turns only about an axis in the
    camera's xy plane.  A prior with a non-finite entry gives (I, 0, (1, 0)).  One track_seed_kernel launch on the
    current stream, no host synchronisation."""
    if not isinstance(refiner, InplaneRefiner):
        raise ValueError("refiner must be a nope_b200.inplane_refine.InplaneRefiner")
    if not torch.is_tensor(R_crop) or R_crop.device.type != "cuda":
        raise _lib.NopeError("seed_centres needs a CUDA tensor (no CPU fallback)")
    if R_crop.dtype not in (torch.float32, torch.float64) or R_crop.dim() < 2 or R_crop.shape[-2:] != (3, 3) or \
            R_crop.numel() == 0:
        raise ValueError(f"R_crop must be float32 or float64 [..., 3, 3], got {R_crop.dtype} {tuple(R_crop.shape)}")
    dev = R_crop.device
    lead = tuple(R_crop.shape[:-2])
    _, tp, _ = refiner._on(dev)
    Rc = R_crop.detach().to(torch.float64).contiguous()
    H = Rc.numel() // 9
    out = {"D": torch.empty(lead + (3, 3), device=dev, dtype=torch.float32),
           "seed": torch.empty(lead, device=dev, dtype=torch.int32),
           "cossin": torch.empty(lead + (2,), device=dev, dtype=torch.float32)}
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_track_seeds(_lib.ptr(Rc), H, _lib.ptr(tp), refiner.num_poses, _lib.ptr(out["D"]),
                                                _lib.ptr(out["seed"]), _lib.ptr(out["cossin"]), _lib.stream(dev)))
    return out


def check_track_args(refiner, all_relativeR, R_prior_crop, k, B, refs=None):
    """ValueError for arguments a tracking step cannot run with, on the host: R_prior_crop [B, P, 3, 3] float32 or
    float64 with 1 <= P <= 16, and check_inplane_refine_args(refiner, all_relativeR, P, k, refs) (refs: the rows
    all_relativeR must have, None for any).  -> P"""
    if not torch.is_tensor(R_prior_crop) or R_prior_crop.dim() != 4 or R_prior_crop.shape[0] != B or \
            R_prior_crop.shape[2:] != (3, 3) or R_prior_crop.shape[1] < 1:
        raise ValueError(f"R_prior [B, P, 3, 3] with B = {B} expected, got "
                         f"{tuple(R_prior_crop.shape) if torch.is_tensor(R_prior_crop) else type(R_prior_crop)}")
    P = int(R_prior_crop.shape[1])
    if P > MAX_KEEP:
        raise ValueError(f"at most {MAX_KEEP} prior rotations per detection, got P = {P}")
    if R_prior_crop.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"R_prior must be float32 or float64, got {R_prior_crop.dtype}")
    check_inplane_refine_args(refiner, all_relativeR, P, k, refs)
    return P


def track_inplane(engine, encoder, ref_feat, crops, all_relativeR, R_prior_crop, refiner, k=5, hidden=None):
    """Refine each crop's roll and viewpoint from prior rotations instead of a search, with any engine that has
    `sweep()`.  ref_feat [B, C, 32, 32], crops [B, 3, 256, 256], all_relativeR [B, N, 6] (the grid of `refiner`), one
    row per detection; R_prior_crop [B, P, 3, 3] (1 <= P <= 16), e.g. the previous frame's rotations in this frame's
    crop camera (crop.to_crop); encoder: a FeatureExtractor on the native engine.  The P priors of each row become
    centres (seed_centres), their latents come from one encode_image_rotated call, and refine_inplane continues from
    them.  -> refine_inplane's dict (D, seed, cossin, score, rel6d, latent [B, k, ...], hypotheses, crops).  Costs P
    * (1 + 2 * steps) encodes and 9 * P * steps hypotheses per row; no host synchronisation.  hidden [B, 256, 256]:
    the crops' masks of pixels that may be hidden, as refine_inplane takes them."""
    if crops.dim() != 4 or tuple(crops.shape[1:]) != (3, 256, 256):
        raise ValueError(f"crops [B, 3, 256, 256] expected, got {tuple(crops.shape)}")
    B = crops.shape[0]
    if ref_feat.dim() != 4 or ref_feat.shape[0] != B:
        raise ValueError(f"ref_feat [B, C, 32, 32] with B = {B} expected, got {tuple(ref_feat.shape)}")
    P = check_track_args(refiner, all_relativeR, R_prior_crop, k, B, B)
    dev = engine.device
    images = crops.to(dev, torch.float32).contiguous()
    cen = seed_centres(R_prior_crop.to(dev), refiner)
    idx = torch.arange(B, device=dev, dtype=torch.int32)[:, None].expand(B, P).reshape(-1)
    lat = encoder.encode_image_rotated(images, idx, cen["cossin"].reshape(B * P, 2))
    return refine_inplane(engine, encoder, ref_feat, images, all_relativeR, cen, lat.view(B, P, *lat.shape[1:]),
                          refiner, k=k, **({} if hidden is None else {"hidden": hidden}))


def _index(rows, device):
    """rows (host ints) as an int64 index on `device`, uploaded from pinned memory without blocking"""
    idx = torch.tensor(rows, dtype=torch.int64)
    return idx.pin_memory().to(device, non_blocking=True) if device.type == "cuda" else idx


def _rows(x, rows, B):
    """x's rows `rows` (host ints) of its B, x itself when rows are all B of them"""
    if x is None or len(rows) == B:
        return x
    return x[_index(rows, x.device)] if torch.is_tensor(x) else x[rows]


def _frame_rows(frame_idx, rows, B):
    """the frame index of detections `rows`: frame_idx None means detection b is in frame b"""
    if frame_idx is None and len(rows) < B:
        return torch.tensor(rows, dtype=torch.int64)
    return _rows(frame_idx, rows, B)


class PoseTracker:
    """Poses of tracked detections, frame after frame (DESIGN.md section 26).

    model: a PoseConditional with the objects' meshes and models_info; bank: a TemplateBank of every object;
    refiner: an InplaneRefiner over the bank's grid.  Each call to step() gives the poses of one frame's detections:
    a track id it has not seen is searched (predict_pose_frames(bank=, refiner=)); a known one is tracked from its
    previous top-`keep` camera rotations (track_pose_frames with R[:, :keep] of the last output, after the contour
    refinement with refine="contour").  A tracked row whose best silhouette IoU over its k hypotheses is below
    `min_iou` (or NaN) is lost: it is searched again in the same frame and its row replaced.  Reading the lost flags
    is one host read of the tracked rows' flags; min_iou = 0 turns the check off and removes that read.  The default
    0.5 is a guess that no real data has checked.  occluders: None or "detections" (each detection's occluders are
    the other detections of its frame, as predict_pose_frames computes them, over all detections of the call).
    occluded_search: the searches and the tracking steps also leave out what those occluders may hide (DESIGN.md
    section 27); it needs occluders="detections"."""

    def __init__(self, model, bank, refiner, keep=2, k=5, min_iou=0.5, refine=None, occluders=None,
                 occluded_search=False):
        from .bank import TemplateBank
        if model.dist is not None:
            raise NotImplementedError("PoseTracker does not shard across GPUs: it runs on one device (unset "
                                      "model.dist)")
        if not isinstance(bank, TemplateBank):
            raise ValueError("bank must be a nope_b200.bank.TemplateBank")
        check_inplane_refine_args(refiner, bank.all_relativeR, keep, k)
        bank.check_grid(refiner.template_poses)
        if k < keep:
            raise ValueError(f"k ({k}) must be at least keep ({keep}): a track keeps its top-keep of k poses")
        if isinstance(min_iou, bool) or not isinstance(min_iou, numbers.Real) or not 0.0 <= min_iou <= 1.0:
            raise ValueError(f"min_iou must be a number in [0, 1], got {min_iou!r}")
        if refine not in (None, "contour"):
            raise ValueError(f"refine must be None or 'contour', got {refine!r}")
        if occluders is not None and not (isinstance(occluders, str) and occluders == "detections"):
            raise ValueError(f"occluders must be None or 'detections', got {occluders!r}")
        if occluded_search and occluders is None:
            raise ValueError("occluded_search=True needs occluders='detections'")
        self.model, self.bank, self.refiner = model, bank, refiner
        self._occluded = {"occluded_search": True} if occluded_search else {}
        self.keep, self.k, self.min_iou = int(keep), int(k), float(min_iou)
        self.refine, self.occluders = refine, occluders
        self.tracks = {}            # track id -> (obj_id, R [keep, 3, 3] float64 on the model's device)

    def reset(self):
        """Forget every track."""
        self.tracks = {}

    def _search(self, frames, masks, K, ids, rows, B, frame_idx, occ):
        return self.model.predict_pose_frames(
            frames, _rows(masks, rows, B), _rows(K, rows, B), [ids[b] for b in rows], k=self.k, refiner=self.refiner,
            refine=self.refine, frame_idx=_frame_rows(frame_idx, rows, B), occluders=_rows(occ, rows, B),
            bank=self.bank, **self._occluded)

    @torch.no_grad()
    def step(self, frames, masks, K, obj_ids, track_ids, frame_idx=None):
        """The poses of B detections: frames, masks, K, obj_ids and frame_idx as predict_pose_frames takes them,
        track_ids B distinct hashable ids (host).  -> predict_pose_frames' dict plus tracked [B] bool (False where the
        row was searched).  Ids absent from the call are forgotten; a known id whose obj_id changed is refused before
        any device work."""
        import numpy as np
        from .crop import _as_numpy, _tensor
        ids = [int(i) for i in np.asarray(obj_ids.detach().cpu() if torch.is_tensor(obj_ids) else obj_ids)
               .reshape(-1).tolist()]
        tids = list(track_ids.tolist() if torch.is_tensor(track_ids) else track_ids)
        B = len(ids)
        if len(tids) != B or len(set(tids)) != B:
            raise ValueError(f"PoseTracker.step: {B} distinct track_ids expected (one per obj_id), got {tids}")
        if masks.shape[0] != B:
            raise ValueError(f"PoseTracker.step: {B} obj_ids for {masks.shape[0]} masks")
        changed = [t for t, i in zip(tids, ids) if t in self.tracks and self.tracks[t][0] != i]
        if changed:
            raise ValueError(f"PoseTracker.step: track ids {changed} changed obj_id (start a new track id)")
        Kh = _as_numpy(K, "K").reshape(-1, 3, 3)
        if len(Kh) not in (1, B):
            raise ValueError(f"K [3, 3] or [B, 3, 3] with B = {B} expected, got {list(Kh.shape)}")
        Kh = np.ascontiguousarray(np.broadcast_to(Kh, (B, 3, 3)))
        fi = None if frame_idx is None else _tensor(frame_idx)
        occ = None
        if self.occluders == "detections":
            from .bop import _to_dev
            from .crop import detection_occluders
            m = _tensor(masks)
            md = m if m.device.type == "cuda" else _to_dev(m, self.model.device, m.dtype)
            occ = detection_occluders(md, frame_idx, num_frames=_tensor(frames).shape[0])
        known = [b for b in range(B) if tids[b] in self.tracks]
        new = [b for b in range(B) if tids[b] not in self.tracks]
        parts = []                                   # (rows, output)
        tracked = [False] * B
        if known:
            prior = torch.stack([self.tracks[tids[b]][1] for b in known])
            out = self.model.track_pose_frames(
                frames, _rows(masks, known, B), Kh[known], [ids[b] for b in known], prior, self.refiner,
                bank=self.bank, k=self.k, refine=self.refine, frame_idx=_frame_rows(fi, known, B),
                occluders=_rows(occ, known, B), **self._occluded)
            lost = []
            if self.min_iou > 0:
                ok = (out["iou"].amax(dim=1) >= self.min_iou).cpu().tolist()    # the one host read per frame
                lost = [b for b, good in zip(known, ok) if not good]
            for b in known:
                tracked[b] = b not in lost
            parts.append((known, out))
            if lost:
                parts.append((lost, self._search(frames, masks, Kh, ids, lost, B, fi, occ)))
        if new:
            parts.append((new, self._search(frames, masks, Kh, ids, new, B, fi, occ)))
        res = dict(parts[0][1]) if len(parts) == 1 else self._merge(parts, B)
        res["tracked"] = torch.tensor(tracked, dtype=torch.bool)
        self.tracks = {tids[b]: (ids[b], res["R"][b, :self.keep]) for b in range(B)}
        return res

    @staticmethod
    def _merge(parts, B):
        """one dict of B rows from the outputs of row subsets, later parts overwriting earlier ones"""
        first = parts[0][1]
        res = {}
        for key, v in first.items():
            res[key] = torch.empty((B,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
        for rows, out in parts:
            for key, v in out.items():
                res[key][_index(rows, v.device)] = v
        return res
