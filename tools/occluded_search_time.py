"""Time the searches under occlusion (DESIGN.md section 27) in ONE process:
  kernels        crop_hidden_kernel for one detection on a 720 x 540 frame, and latent_visibility_kernel for that
                 detection's A = 36 rolled copies (the maps of an in-plane or bank search), each alone;
  predict_pose   N = 642 poses, Q = 1 and 16 queries, with an all-zero hidden= (the visible sweep and its maps)
                 against none (the sweep without maps);
  frames         predict_pose_frames(bank=, occluders="detections") of tools/bank_time.py's six-detection frame (a
                 bank of the six objects at N = 642, A = 36), with occluded_search on and off.
    python tools/occluded_search_time.py --reps 7 --out /tmp/occluded.json

Accuracy (--standin queries, seeded weights): the render engine of tools/inplane_refine_time.py (three boxes, level-2
grid, seeded template encoder) with its 642 template latents materialised once; queries are renders at seeded
viewpoints and rolls.  A nearer sphere -- a disc in the 256 x 256 render -- is moved from the silhouette's box centre
along a seeded direction until it hides 20 / 40 / 60 % of the silhouette (bisection; the median cover reached is
reported); the hidden object pixels are set to -1 (background) and `hidden` is the disc.  retrieval_inplane's stages
at A = 36 (encode_image_inplane, latent_visibility, nope_score_topk_visible; nope_score_topk_multi without hidden)
score every query; the table is the median / p90 top-1 geodesic error for l2 and cosine_occlusion, each with and
without hidden.  --margins also dilates the maps by 1, 2, ... latent pixels (a max-pool here, outside the kernel) to
measure whether hiding the neighbours that the encoder's receptive field mixes in would help.
This describes the seeded encoder on renders; it says nothing about trained weights.
Device events around whole calls, warm-up of every shape, the cases alternated inside each repetition; ms is the
median over repetitions with the min / max beside it.  Prints the card name and power limit with the numbers.
Seeded weights: the times do not depend on them.  A development aid, not the bench."""
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
from nope_b200.inplane import inplane_table
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
from nope_b200.visibility import crop_hidden, latent_visibility

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def disc_cover(S, cover, rng, radius):
    """a disc of `radius` px moved from the box centre of silhouette S [256, 256] (bool) along a seeded direction
    until it covers `cover` of S (bisection on the distance) -> (disc [256, 256] bool, achieved cover)"""
    ys, xs = torch.nonzero(S, as_tuple=True)
    n = float(S.sum())
    v0, u0 = (float(ys.min()) + float(ys.max())) / 2, (float(xs.min()) + float(xs.max())) / 2
    a = rng.uniform(0, 2 * math.pi)
    yy, xx = torch.meshgrid(torch.arange(256.0, device=S.device), torch.arange(256.0, device=S.device), indexing="ij")

    def place(d):
        disc = (yy - (v0 + d * math.sin(a))) ** 2 + (xx - (u0 + d * math.cos(a))) ** 2 < radius * radius
        return disc, float((disc & S).sum()) / n
    lo, hi = 0.0, 3.0 * radius + 128.0
    for _ in range(20):
        mid = 0.5 * (lo + hi)
        if place(mid)[1] > cover:
            lo = mid
        else:
            hi = mid
    return place(0.5 * (lo + hi))


def accuracy(model, n_q, info, A=36, covers=(0.2, 0.4, 0.6), margins=(0, 1, 2), seed=3):
    """the stand-in table: one JSON line per (cover, metric, hidden, margin)"""
    from inplane_refine_time import RenderEngine, geodesic_deg, three_boxes
    from nope_b200.inplane import inplane_rotations
    from nope_b200.model import _score_multi, topk
    from nope_b200.poses import relative_rotation_6d, viewpoint_rotations
    from nope_b200.visibility import latent_visibility_inplane, score_visible
    from nope_b200.vsd import Mesh
    enc = model.u_net.encoder
    R2 = icosphere_object_rotations(2)
    ref_R = R2[7]
    eng = RenderEngine(enc, Mesh(*three_boxes()), ref_R)
    rel = relative_rotation_6d(R2, ref_R)[None].cuda()
    t = eng.templates(rel).view(1, 642, enc.latent_dim, 32, 32).contiguous()        # materialised once
    rng = np.random.default_rng(seed)
    gamma = rng.uniform(-math.pi, math.pi, n_q)
    Rz = np.stack([[[math.cos(x), -math.sin(x), 0], [math.sin(x), math.cos(x), 0], [0, 0, 1]] for x in gamma])
    qR = torch.from_numpy(Rz @ viewpoint_rotations(rng.standard_normal((n_q, 3)))).cuda()
    clean = eng.images(qR)
    tp = torch.from_numpy(R2).cuda()
    Rzs = inplane_rotations(A).cuda()
    slots = torch.zeros(1, device="cuda", dtype=torch.int32)
    row_off = torch.tensor([0, n_q * A], device="cuda", dtype=torch.int32)
    lines = []
    for cover in covers:
        hidden = torch.zeros((n_q, 256, 256), dtype=torch.bool, device="cuda")
        achieved = []
        for i in range(n_q):
            S = clean[i, 0] > -1.0
            radius = math.sqrt(float(S.sum()) / math.pi)                    # about as large as the object
            hidden[i], c = disc_cover(S, cover, rng, radius)
            achieved.append(c)
        q_img = torch.where(hidden[:, None] & (clean > -1.0), torch.full_like(clean, -1.0), clean)
        lat = enc.encode_image_inplane(q_img, A)                            # [n, A, C, 32, 32]
        for metric in ("l2", "cosine_occlusion"):
            thr = model._occlusion_threshold()
            runs = [("none", None)] + [("hidden", m) for m in margins]
            for name, margin in runs:
                if margin is None:
                    sim, _, _ = _score_multi(lat.reshape(1, n_q * A, *lat.shape[2:]).contiguous(), t, 1, n_q * A,
                                             metric, thr)
                else:
                    vis = latent_visibility_inplane(hidden, A).reshape(n_q * A, 1, 32, 32)
                    if margin:                              # hidden blocks dilated by `margin` latent pixels
                        hid = torch.nn.functional.max_pool2d(1.0 - vis.float(), 2 * margin + 1, 1, margin)
                        vis = (hid == 0).to(torch.uint8)
                    vis = vis.reshape(n_q * A, 32, 32)
                    sim, _ = score_visible(lat.reshape(n_q * A, *lat.shape[2:]), t, slots, row_off, A, vis, metric,
                                           thr, 0)
                _, flat = topk(sim.view(n_q, A * 642), 1)
                n, a = flat[:, 0] % 642, flat[:, 0] // 642
                err = geodesic_deg(Rzs[a] @ tp[n], qR)
                lines.append({"case": "standin", "cover": cover, "cover_achieved_median": round(
                    statistics.median(achieved), 3), "metric": metric, "hidden": name != "none", "margin": margin,
                    "median_deg": round(float(err.median()), 2), "p90_deg": round(float(err.quantile(0.9)), 2),
                    "queries": n_q, "angles": A, **info})
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--angles", type=int, default=36)
    ap.add_argument("--reps", type=int, default=7, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=3, help="calls per timed window (x 100 for the kernels)")
    ap.add_argument("--standin", type=int, default=64, help="queries of the accuracy stand-in (0: skip it)")
    ap.add_argument("--margins", type=int, nargs="+", default=[0, 1, 2], help="dilations of the stand-in's maps")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("occluded_search_time.py needs a CUDA device")

    info = card()
    dev = "cuda:0"
    model = build_model(device=dev).load_state_dict(weights.make_full_state_dict(seed=0)).eval()
    rel = synthetic_pose_batch(642, 1)[0].to(dev)
    tp = torch.from_numpy(icosphere_object_rotations(2)).to(dev)
    g = torch.Generator().manual_seed(0)
    ref = (torch.rand(1, 3, 256, 256, generator=g) * 2 - 1).to(dev)
    Qmax = max(args.queries)
    qry = (torch.rand(Qmax, 3, 256, 256, generator=g) * 2 - 1).to(dev)
    zeros = torch.zeros(Qmax, 256, 256, dtype=torch.uint8, device=dev)

    # one detection: a 720 x 540 frame whose left half may hide the object, a crop map of a 2x magnification
    occ = torch.zeros(1, 540, 720, dtype=torch.uint8, device=dev)
    occ[:, :, :360] = 1
    inv = torch.tensor([[[0.5, 0.0, 296.0], [0.0, 0.5, 206.0], [0.0, 0.0, 1.0]]], dtype=torch.float64)
    hidden = crop_hidden(occ, inv)
    A = args.angles
    cs = inplane_table(A).to(dev)
    idx = torch.zeros(A, dtype=torch.int32, device=dev)

    # tools/bank_time.py's frame: six 78 mm boxes, one per object, and a bank of the six objects
    from bank_time import K3, scene
    from nope_b200 import bop
    mesh, diameter, ids, masks, frames, fidx = scene(1, 6)
    minfo = {"diameter": diameter, "symmetries_discrete": [], "symmetries_continuous": []}
    for i in range(1, 7):
        model.tless_cad[i] = mesh
        model.bop_models[i] = {"diameter": diameter, "symmetries": bop.symmetry_transformations(minfo), "info": minfo}
    bank = model.build_template_bank(list(range(1, 7)), (torch.rand(6, 3, 256, 256, generator=g) * 2 - 1).to(dev),
                                     synthetic_pose_batch(642, 6)[0].to(dev), tp.cpu())

    def frame(on):
        return lambda: model.predict_pose_frames(frames, masks, K3, ids, angles=A, k=5, frame_idx=fidx,
                                                 occluders="detections", bank=bank, occluded_search=on)

    fns = {("crop_hidden", 1): lambda: crop_hidden(occ, inv),
           ("frames_bank", 6): frame(False), ("frames_bank_occluded_search", 6): frame(True),
           ("latent_visibility", A): lambda: latent_visibility(hidden, cs, idx)}
    for Q in args.queries:
        fns[("predict_pose", Q)] = lambda Q=Q: model.predict_pose(qry[:Q], ref, rel, tp, k=5)
        fns[("predict_pose_hidden", Q)] = lambda Q=Q: model.predict_pose(qry[:Q], ref, rel, tp, k=5,
                                                                         hidden=zeros[:Q])
    for fn in fns.values():                        # warm every shape
        fn()
        fn()
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for key, fn in fns.items():
            n = args.iters * (100 if key[0] in ("crop_hidden", "latent_visibility") else 1)
            samples[key].append(timed_ms(fn, n))

    lines = []
    if args.standin:
        lines += accuracy(model, args.standin, info, margins=tuple(args.margins))
    for (name, n), ms in samples.items():
        row = {"case": name, "n": n, "ms": round(statistics.median(ms), 4), "ms_min": round(min(ms), 4),
               "ms_max": round(max(ms), 4)}
        if name == "predict_pose_hidden":
            row["extra_ms_over_predict_pose"] = round(row["ms"] - statistics.median(samples[("predict_pose", n)]), 4)
        if name == "frames_bank_occluded_search":
            row["extra_ms_over_frames_bank"] = round(row["ms"] - statistics.median(samples[("frames_bank", n)]), 4)
        lines.append({**row, **info})
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
