"""Time pose tracking (DESIGN.md section 26) against the per-frame searches, and measure all three on a render-based
stand-in, in ONE process.

Time per frame: the synthetic scene of bank_time.py (D detections of a 78 mm box per 720 x 540 frame, one per object,
Primesense intrinsics), turned into sequences in which each object turns --delta degrees per frame about its own
seeded axis; the level-2 grid (N = 642), A = 36, a template bank of the D objects, the fp16 UNet and encoder.
  track          PoseTracker.step on frames 1 ... F-1 after a first frame (min_iou = 0: every row tracked, no re-search)
  bank           predict_pose_frames(bank=) on the same frames
  bank_refined   predict_pose_frames(bank=, refiner=) (keep = 2, 4 steps)
for keep in --keeps and steps in --steps of the tracker.  Device events around whole calls after a warm-up, the
paths alternated inside each repetition; ms is the median over repetitions with min / max.

Accuracy (seeded weights, a stand-in): the RenderEngine of inplane_refine_time.py (templates are encoder latents of
renders of three boxes at the relative pose).  --sequences trajectories of --length frames start at seeded
viewpoints and rolls and turn by delta degrees per frame in viewpoint (about a seeded axis in the camera's xy plane)
and delta in roll, for delta in --deltas.  Reports the median / p90 geodesic error of the tracker (frame 0 the refined
search, then track_inplane from the previous frame's top-keep rotations), the per-frame in-plane search and the
per-frame refined search, and the share of frame-to-frame motions outside the refinement's reach: at least 2 theta0
about x or y, or 2 phi0 about z (computed from the trajectory, not measured).  These figures describe the seeded
encoder on renders; they say nothing about trained weights.

Prints the card name and power limit with the numbers.  A development aid, not the bench.
    python tools/track_time.py --out /tmp/track.json"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import bop
from nope_b200 import synth_weights as weights
from nope_b200.inplane import inplane_rotations
from nope_b200.inplane_refine import InplaneRefiner, pose_rotations, refine_inplane
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d, synthetic_pose_batch, \
    viewpoint_rotations
from nope_b200.refine import axis_angle_matrix
from nope_b200.track import PoseTracker, track_inplane
from nope_b200.vsd import Mesh, render_depth
from oracle import render_oracle as ro

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bank_time import K3, H, W, stats                                    # noqa: E402
from inplane_refine_time import RenderEngine, geodesic_deg, three_boxes  # noqa: E402
from multi_query_time import card, timed_ms                             # noqa: E402


def sequences(F, D, delta, seed=0):
    """F frames of D boxes, box j turning delta degrees per frame about its own seeded axis at a fixed position ->
    (mesh, diameter, masks [F, D, H, W] uint8 CUDA, frames [F, H, W, 3] uint8 CUDA)"""
    v, f = ro.box()
    mesh = Mesh(v, f)
    diameter = float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))
    rng = np.random.default_rng(seed)
    poses = []
    for j in range(D):
        R0 = ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        u, v_, z = (j + 0.5) * W / D, rng.uniform(150, H - 150), rng.uniform(600.0, 900.0)
        poses.append((R0, axis, np.linalg.solve(K3, [u, v_, 1.0]) * z))
    masks = torch.empty((F, D, H, W), dtype=torch.uint8, device="cuda")
    for fr in range(F):
        for j, (R0, axis, t) in enumerate(poses):
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = axis_angle_matrix(math.radians(delta * fr) * axis) @ R0, t
            masks[fr, j] = (render_depth(mesh, torch.from_numpy(T), K3, (H, W))[0] > 0).to(torch.uint8) * 255
    frames = masks.amax(1)[..., None].expand(F, H, W, 3).contiguous()
    return mesh, diameter, masks, frames


def timing(model, args, info, emit):
    F, D = args.frames, args.detections
    mesh, diameter, masks, frames = sequences(F, D, args.delta)
    ids = list(range(1, D + 1))
    minfo = {"diameter": diameter, "symmetries_discrete": [], "symmetries_continuous": []}
    for i in ids:
        model.tless_cad[i] = mesh
        model.bop_models[i] = {"diameter": diameter, "symmetries": bop.symmetry_transformations(minfo), "info": minfo}
    tp = torch.from_numpy(icosphere_object_rotations(2))
    g = torch.Generator().manual_seed(1)
    refs = (torch.rand(D, 3, 256, 256, generator=g) * 2 - 1).cuda()
    bank = model.build_template_bank(ids, refs, synthetic_pose_batch(642, D)[0].cuda(), tp)
    searched = InplaneRefiner(tp, angles=36, steps=4)
    fi = torch.zeros(D, dtype=torch.int64)
    one = lambda fr: (frames[fr:fr + 1], masks[fr], K3, ids)                     # noqa: E731
    paths = {"bank": lambda fr: model.predict_pose_frames(*one(fr), k=5, frame_idx=fi, bank=bank),
             "bank_refined": lambda fr: model.predict_pose_frames(*one(fr), k=5, refiner=searched, frame_idx=fi,
                                                                  bank=bank)}
    trackers = {}
    for steps in args.steps:
        ref = InplaneRefiner(tp, angles=36, steps=steps)
        for keep in args.keeps:
            tr = PoseTracker(model, bank, ref, keep=keep, k=5, min_iou=0.0)
            tr.step(*one(0), ids, frame_idx=fi)
            trackers[(keep, steps)] = tr
            paths[f"track keep={keep} steps={steps}"] = \
                lambda fr, tr=tr: tr.step(*one(fr), ids, frame_idx=fi)
    for fn in paths.values():
        fn(1)                                                                      # warm-up of every shape
    times = {name: [] for name in paths}
    for _ in range(args.reps):
        per = {name: 0.0 for name in paths}
        for fr in range(1, F):
            for name, fn in paths.items():
                per[name] += timed_ms(lambda: fn(fr), 1)
        for name in paths:
            times[name].append(per[name] / (F - 1))
    for name, t in times.items():
        rec = {"case": name, "frames": F - 1, "detections_per_frame": D, "delta_deg": args.delta, "angles": 36,
               "poses": 642, "per_frame": stats(t), "per_detection_ms": round(stats(t)["ms"] / D, 3)}
        if name.startswith("track"):
            keep, steps = (int(s.split("=")[1]) for s in name.split()[1:])
            rec.update(encodes_per_detection=keep * (1 + 2 * steps), hypotheses_per_detection=9 * keep * steps)
        elif name == "bank_refined":
            rec.update(encodes_per_detection=36 + searched.crops(2), hypotheses_per_detection=searched.hypotheses(2))
        else:
            rec.update(encodes_per_detection=36, hypotheses_per_detection=0)
        emit(rec)


def rz(t):
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def accuracy(model, args, emit):
    enc = model.u_net.encoder
    R2 = icosphere_object_rotations(2)
    ref_R = R2[7]
    eng = RenderEngine(enc, Mesh(*three_boxes()), ref_R)
    A, keep, steps, S, L = 36, 2, 4, args.sequences, args.length
    ir = InplaneRefiner(R2, angles=A, steps=steps)
    reach_xy, reach_z = 2 * ir.theta0, 2 * ir.phi0
    tp = torch.from_numpy(R2).cuda()
    Rzs = inplane_rotations(A).cuda()
    rel1 = relative_rotation_6d(R2, ref_R)[None].cuda()
    for delta in args.deltas:
        rng = np.random.default_rng(int(delta * 10))
        d = math.radians(delta)
        V0 = viewpoint_rotations(rng.standard_normal((S, 3)))
        g0 = rng.uniform(-math.pi, math.pi, S)
        axes = rng.standard_normal((S, 2))
        axes /= np.linalg.norm(axes, axis=1, keepdims=True)
        qR = np.stack([[rz(g0[s] + t * d) @ axis_angle_matrix(t * d * np.array([*axes[s], 0.0])) @ V0[s]
                        for t in range(L)] for s in range(S)])                   # [S, L, 3, 3]
        # the frame-to-frame motion in the camera frame, against the refinement's reach
        M = np.einsum("slij,slkj->slik", qR[:, 1:], qR[:, :-1])
        w = np.stack([M[..., 2, 1] - M[..., 1, 2], M[..., 0, 2] - M[..., 2, 0], M[..., 1, 0] - M[..., 0, 1]], -1)
        ang = np.arccos(np.clip((np.trace(M, axis1=-2, axis2=-1) - 1) / 2, -1, 1))
        w = w / np.maximum(2 * np.sin(ang), 1e-300)[..., None] * ang[..., None]
        outside = float(((np.abs(w[..., 0]) >= reach_xy) | (np.abs(w[..., 1]) >= reach_xy) |
                         (np.abs(w[..., 2]) >= reach_z)).mean())
        qRt = torch.from_numpy(qR.reshape(S * L, 3, 3)).cuda()
        imgs = eng.images(qRt)                                                       # [S * L, 3, 256, 256]
        n_q = S * L
        qf = enc.encode_image_inplane(imgs, A)
        rf1 = torch.zeros(1, enc.latent_dim, 32, 32, device=qf.device)
        sim = eng.sweep(rf1, rel1, qf.view(1, n_q * A, *qf.shape[2:]))["sim"].view(n_q, A * 642)
        flat = torch.sort(-sim, dim=1, stable=True).indices[:, :keep]
        n, a = flat % 642, flat // 642
        err = {"inplane": geodesic_deg(Rzs[a[:, 0]] @ tp[n[:, 0]], qRt)}
        lat = qf[torch.arange(n_q, device=qf.device)[:, None], a]
        out = refine_inplane(eng, enc, rf1, imgs[None], rel1, (n[None], a[None]), lat[None], ir, k=keep)
        Rref = pose_rotations(out["D"], out["seed"], out["cossin"], ir)[0]              # [n_q, keep, 3, 3]
        err["inplane_refined"] = geodesic_deg(Rref[:, 0], qRt)
        # the tracker: frame 0 from the refined search, then track_inplane on each sequence's next frame
        rfS, relS = rf1.expand(S, *rf1.shape[1:]), rel1.expand(S, 642, 6)
        imgs = imgs.view(S, L, 3, 256, 256)
        prior = Rref.view(S, L, keep, 3, 3)[:, 0]
        tracked = [prior[:, 0]]
        for t in range(1, L):
            o = track_inplane(eng, enc, rfS, imgs[:, t], relS, prior, ir, k=keep)
            prior = pose_rotations(o["D"], o["seed"], o["cossin"], ir)
            tracked.append(prior[:, 0])
        err["track"] = geodesic_deg(torch.stack(tracked, 1).reshape(n_q, 3, 3), qRt)
        for name, e in err.items():
            e = e.view(S, L)[:, 1:].reshape(-1)                                       # frames 1 ... L-1
            emit({"case": f"standin {name}", "delta_deg": delta, "sequences": S, "frames": L - 1, "keep": keep,
                  "steps": steps, "median_deg": round(float(e.median()), 3),
                  "p90_deg": round(float(e.quantile(0.9)), 3),
                  "outside_reach": round(outside, 3), "reach_xy_deg": round(math.degrees(reach_xy), 3),
                  "reach_roll_deg": round(math.degrees(reach_z), 3)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--detections", type=int, default=6)
    ap.add_argument("--delta", type=float, default=2.0, help="degrees per frame of the timing sequences")
    ap.add_argument("--keeps", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--deltas", type=float, nargs="+", default=[1.0, 2.0, 4.0])
    ap.add_argument("--sequences", type=int, default=8)
    ap.add_argument("--length", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_time.py needs a CUDA device")
    info = card()
    model = build_model(device="cuda:0", precision="fp16").load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    lines = []

    def emit(rec):
        rec.update(info)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    with torch.no_grad():
        timing(model, args, info, emit)
        accuracy(model, args, emit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
