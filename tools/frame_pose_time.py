"""Time predict_pose_frames (DESIGN.md section 23) and its stages in ONE process, for B detections in B 720 x 540
Primesense frames (a 78 mm box rendered at seeded poses), A = 36 in-plane angles, the level-2 grid (N = 642), the
fp16 UNet and the fp16 template encoder:
  frames_total      predict_pose_frames, refine=None
  crop              frame_crops: initial_translation, the one copy of t0, crop_transforms (cv2), crop_frames,
                    crop_camera
  encoders          the reference's encode_image plus encode_image_inplane of the B crops at A angles
  search            predict_pose_inplane (encoders + sweep + ranking); sweep = search - encoders
  to_camera         the re-expression of the B x 5 rotations
  translation       estimate_translation of the B x 5 hypotheses (4 updates)
  kernels           nope_crop_camera + nope_crop_rotate alone (device events over --kernel-iters calls)
Device events around whole calls after a warm-up; the median over --reps with min / max.  Seeded weights.  Prints
one JSON line per case with the card name and power limit read in the same run.
    python tools/frame_pose_time.py --reps 5 --out /tmp/frame_pose.json
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

from nope_b200 import synth_weights as weights
from nope_b200 import translation
from nope_b200.crop import _camera, frame_crops, to_camera
from nope_b200.encoder import FeatureExtractor
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d
from nope_b200.vsd import Mesh, render_depth
from oracle import render_oracle as ro

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402

K3 = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]])
H, W = 540, 720


def scene(mesh, B, seed=0):
    rng = np.random.default_rng(seed)
    masks = []
    while len(masks) < B:
        T = np.eye(4)
        T[:3, :3] = ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3]
        T[:3, 3] = np.linalg.solve(K3, [rng.uniform(80, W - 80), rng.uniform(80, H - 80), 1.0]) * rng.uniform(500, 1100)
        m = render_depth(mesh, torch.from_numpy(T), K3, (H, W))[0] > 0
        if m.any():
            masks.append(m.to(torch.uint8) * 255)
    masks = torch.stack(masks)
    return masks[..., None].expand(B, H, W, 3).contiguous(), masks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--detections", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--angles", type=int, default=36)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_pose_time.py needs a CUDA device")
    info = card()
    A, k = args.angles, 5
    full = weights.make_full_state_dict(seed=0)
    model = build_model(device="cuda:0").load_state_dict(full).eval()
    fe = FeatureExtractor(descriptor_size=8, precision="fp16").cuda()
    fe.load_state_dict({key[len("encoder."):]: v for key, v in full.items()
                        if key.startswith("encoder.backbone.") or key.startswith("encoder.projector.")})
    model.u_net.encoder = fe
    v, f = ro.box()
    mesh = Mesh(v, f)
    d = float(np.linalg.norm([60.0, 40.0, 30.0]))
    model.tless_cad[1] = mesh
    model.bop_models[1] = {"diameter": d}
    R2 = icosphere_object_rotations(2)
    rel = relative_rotation_6d(R2, R2[7])[None].cuda()
    tp = torch.from_numpy(R2).cuda()
    g = torch.Generator().manual_seed(0)
    ref = (torch.rand(1, 3, 256, 256, generator=g) * 2 - 1).cuda()

    lines = []
    with torch.no_grad():
        for B in args.detections:
            frames, masks = scene(mesh, B, seed=B)
            dd = np.full(B, d)
            crops, t0, Rv, _ = frame_crops(frames, masks, K3, dd)
            R_crop = model.predict_pose_inplane(crops, ref, rel, tp, k=k, angles=A)[0]
            R = to_camera(R_crop, Rv)
            Kb = np.broadcast_to(K3, (B, 3, 3)).copy()
            pose = np.tile(np.eye(4), (B, 1, 1))
            pose[:, :3, 3] = t0.cpu().numpy()
            cases = {
                "frames_total": lambda: model.predict_pose_frames(frames, masks, K3, [1] * B, ref, rel, tp,
                                                                  angles=A, k=k),
                "crop": lambda: frame_crops(frames, masks, K3, dd),
                "encoders": lambda: (fe.encode_image(ref), fe.encode_image_inplane(crops, A)),
                "search": lambda: model.predict_pose_inplane(crops, ref, rel, tp, k=k, angles=A),
                "to_camera": lambda: to_camera(R_crop, Rv),
                "translation": lambda: translation.estimate_translation(mesh, R, Kb, masks, t_init=t0),
            }
            for fn in cases.values():
                fn()
                fn()
            samples = {name: [] for name in cases}
            for _ in range(args.reps):
                for name, fn in cases.items():
                    samples[name].append(timed_ms(fn, 1))
            samples["kernels"] = [timed_ms(lambda: (to_camera(R_crop, _camera(pose, True, Rv.device))),
                                           args.kernel_iters) for _ in range(args.reps)]
            med = {name: statistics.median(ms) for name, ms in samples.items()}
            for name, ms in samples.items():
                lines.append({"case": name, "B": B, "A": A, "N": 642, "ms": round(med[name], 3),
                              "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), "reps": len(ms), **info})
            lines.append({"case": "split", "B": B, "crop_ms": round(med["crop"], 3),
                          "encoders_ms": round(med["encoders"], 3),
                          "sweep_ms": round(med["search"] - med["encoders"], 3),
                          "translation_ms": round(med["translation"], 3), "total_ms": round(med["frames_total"], 3),
                          "crop_camera_and_rotate_ms": round(med["kernels"], 4), **info})
    torch.cuda.synchronize()
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
