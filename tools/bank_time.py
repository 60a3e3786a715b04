"""Time template banks (DESIGN.md section 25) on a synthetic T-LESS-like scene, in ONE process: F frames (720 x 540,
Primesense intrinsics) with D detections each, one per object of O objects (a 78 mm box rendered at seeded poses),
A = 36 in-plane angles, the level-2 grid (N = 642) and, for the bank search, also the level-3 grid (N = 2562); the fp16
UNet and the fp16 template encoder.
  build               build_template_bank of the O objects (one encoder call, one sweep), per object
  bank_search         predict_pose_bank of all F * D crops, per detection
  sweep_search        predict_pose_inplane of the same crops with reference[slot] (a sweep per detection), per
                      detection
  encode_floor        encode_image_inplane of the crops alone, per detection: what a bank search cannot go below
  frames_bank         predict_pose_frames(bank=) of the F frames, per frame
  frames_references   predict_pose_frames with the references, per frame
The two searches and the two frame paths alternate inside each repetition; the median over --reps with min / max.
Device events around whole calls after a warm-up.  Also prints the bank's memory, and the card name and power limit
read in the same run.  Seeded weights: the times do not depend on them.
    python tools/bank_time.py --reps 3 --out /tmp/bank.json
A development aid, not the bench."""
import argparse
import json
import math
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import bop
from nope_b200 import synth_weights as weights
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
from nope_b200.vsd import Mesh, render_depth
from oracle import render_oracle as ro

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402

K3 = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]])
H, W = 540, 720


def scene(F, D, seed=0):
    """F frames with D detections each (detection j of a frame is object j + 1) -> (mesh, diameter, ids, masks [F * D,
    H, W] uint8 CUDA, frames [F, H, W, 3] uint8 CUDA, frame_idx [F * D])"""
    v, f = ro.box()
    mesh = Mesh(v, f)
    diameter = float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))
    rng = np.random.default_rng(seed)
    masks, ids, fidx = [], [], []
    for fr in range(F):
        for j in range(D):
            while True:
                R = ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)
                u, v_, z = rng.uniform(100, W - 100), rng.uniform(100, H - 100), rng.uniform(500.0, 1000.0)
                T = np.eye(4)
                T[:3, :3], T[:3, 3] = R, np.linalg.solve(K3, [u, v_, 1.0]) * z
                m = render_depth(mesh, torch.from_numpy(T), K3, (H, W))[0] > 0
                if bool(m.any()):
                    break
            masks.append(m.to(torch.uint8) * 255)
            ids.append(j + 1)
            fidx.append(fr)
    masks = torch.stack(masks)
    frames = torch.stack([masks[fr * D:(fr + 1) * D].amax(0) for fr in range(F)])
    frames = frames[..., None].expand(F, H, W, 3).contiguous()
    return mesh, diameter, ids, masks, frames, torch.tensor(fidx)


def stats(xs):
    return {"ms": round(statistics.median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--detections", type=int, default=6, help="detections per frame, one per object")
    ap.add_argument("--angles", type=int, default=36)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bank_time.py needs a CUDA device")
    info = card()
    model = build_model(device="cuda:0", precision="fp16").load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    F, O, A = args.frames, args.detections, args.angles
    mesh, diameter, ids, masks, frames, fidx = scene(F, O)
    Bd = len(ids)
    obj_ids = list(range(1, O + 1))
    minfo = {"diameter": diameter, "symmetries_discrete": [], "symmetries_continuous": []}
    for i in obj_ids:
        model.tless_cad[i] = mesh
        model.bop_models[i] = {"diameter": diameter, "symmetries": bop.symmetry_transformations(minfo), "info": minfo}
    g = torch.Generator().manual_seed(1)
    refs = (torch.rand(O, 3, 256, 256, generator=g) * 2 - 1).cuda()
    slots = [i - 1 for i in ids]
    grids = {}
    for level in (2, 3):
        tp = torch.from_numpy(icosphere_object_rotations(level))
        grids[tp.shape[0]] = (synthetic_pose_batch(tp.shape[0], O)[0].cuda(), tp)
    lines = []

    def emit(rec):
        rec.update(info)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    # ---------------------------------------------------------------- build, per object
    banks = {}
    for N, (rel, tp) in grids.items():
        banks[N] = model.build_template_bank(obj_ids, refs, rel, tp)           # warm-up, kept
        t = [timed_ms(lambda: model.build_template_bank(obj_ids, refs, rel, tp), 1) / O for _ in range(args.reps)]
        b = banks[N]
        emit({"case": "build", "poses": N, "objects": O, "per_object": stats(t),
              "bank_MiB": round(b.nbytes / 2 ** 20, 2),
              "templates_MiB_per_object": round(b.templates[0].numel() * 4 / 2 ** 20, 2),
              "KiB_per_template": b.templates[0, 0].numel() * 4 / 1024})

    # ---------------------------------------------------------------- searches, per detection
    from nope_b200.crop import frame_crops
    crops, _, _, _ = frame_crops(frames, masks, K3, np.full(Bd, diameter), frame_idx=fidx)
    rel, tp = grids[642]
    ref_d, rel_d, tp_d = refs[slots], rel[slots], tp.cuda()
    enc = model.u_net.encoder
    paths = {"bank_search": lambda: model.predict_pose_bank(crops, ids, banks[642], k=5, angles=A),
             "sweep_search": lambda: model.predict_pose_inplane(crops, ref_d, rel_d, tp_d, k=5, angles=A),
             "encode_floor": lambda: enc.encode_image_inplane(crops, A),
             "bank_search_2562": lambda: model.predict_pose_bank(crops, ids, banks[2562], k=5, angles=A)}
    for fn in paths.values():
        fn()
    times = {name: [] for name in paths}
    for _ in range(args.reps):
        for name, fn in paths.items():
            times[name].append(timed_ms(fn, 1) / Bd)
    _, n_b, a_b, sim_b = paths["bank_search"]()
    _, n_s, a_s, sim_s = paths["sweep_search"]()
    agree = float(((n_b == n_s) & (a_b == a_s)).all(1).float().mean())
    rel_err = float(((sim_b - sim_s).abs() / sim_s.abs().clamp_min(1e-30)).max())
    for name, t in times.items():
        emit({"case": name, "detections": Bd, "angles": A, "poses": 2562 if name.endswith("2562") else 642,
              "per_detection": stats(t)})
    emit({"case": "bank_vs_sweep", "top_k_rows_equal": agree, "score_max_rel": rel_err})

    # ---------------------------------------------------------------- frames, per frame
    fpaths = {"frames_bank": lambda: model.predict_pose_frames(frames, masks, K3, ids, angles=A, k=5, frame_idx=fidx,
                                                               bank=banks[642]),
              "frames_references": lambda: model.predict_pose_frames(frames, masks, K3, ids, ref_d, rel_d, tp_d,
                                                                     angles=A, k=5, frame_idx=fidx)}
    for fn in fpaths.values():
        fn()
    ftimes = {name: [] for name in fpaths}
    for _ in range(args.reps):
        for name, fn in fpaths.items():
            ftimes[name].append(timed_ms(fn, 1) / F)
    for name, t in ftimes.items():
        emit({"case": name, "frames": F, "detections_per_frame": O, "angles": A, "poses": 642,
              "per_frame": stats(t)})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
