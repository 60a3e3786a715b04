"""Time off-grid pose refinement against the grid searches over the synthetic icospheres, for one reference and Q
query images, in ONE process:
  exhaustive   predict_pose over level 3 (2562 poses) and over level 2 (642 poses, the refinement's seed sweep);
  c2f 2->3     predict_pose_coarse_to_fine over levels 2, 3 with keep 8;
  refine       predict_pose_refined from level 2 (642 poses) with keep in --keeps and --steps steps.
    python tools/refine_time.py --queries 1 16 --reps 5 --out /tmp/refine.json
Device events around whole calls (encoder included), warm-up of every shape, the cases alternated inside each
repetition; ms is the median over repetitions with the min / max beside it.  `hypotheses` is what one call sweeps.

The top-1 geodesic error (median / p90, degrees) is measured on features, not images: --standin seeded off-grid
viewpoints (the camera at a random point of the sphere, the grids' up-vector rule), each query feature the engine's
own template there.  No trained checkpoint exists, so the figure describes the seeded weights' score landscape,
nothing about trained weights.  Prints the card name and power limit with the numbers.  A development aid, not the
bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import synth_weights as weights
from nope_b200.hierarchy import PoseHierarchy, search
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d, viewpoint_rotations
from nope_b200.refine import PoseRefiner, refine, template_rotations

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def geodesic_deg(A, B):
    t = (A.double() * B.double()).sum(dim=(-2, -1))
    return torch.rad2deg(torch.arccos(((t - 1) / 2).clamp(-1, 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--keeps", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=3, help="calls per timed window")
    ap.add_argument("--standin", type=int, default=64, help="seeded off-grid queries for the geodesic error")
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0", precision=args.precision).load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    Rl = {l: icosphere_object_rotations(l) for l in (2, 3)}
    ref_R = Rl[3][7]
    rel = {l: relative_rotation_6d(Rl[l], ref_R)[None].cuda() for l in Rl}
    tposes = torch.from_numpy(Rl[3])
    hier = PoseHierarchy([Rl[2], Rl[3]])
    refiner = PoseRefiner(Rl[2], steps=args.steps)
    # (name, level) for the exhaustive sweeps, (name, keep) for the others
    cases = [("exhaustive", 3), ("exhaustive", 2), ("c2f 2->3", 8)] + [("refine", k) for k in args.keeps]

    g = torch.Generator().manual_seed(0)
    ref = torch.rand(1, 3, 256, 256, generator=g).cuda()
    qry = torch.rand(max(args.queries), 3, 256, 256, generator=g).cuda()

    def call(case, Q):
        name, keep = case
        if name == "exhaustive":
            return lambda: model.predict_pose(qry[:Q], ref, rel[keep], torch.from_numpy(Rl[keep]), k=5)
        if name == "c2f 2->3":
            return lambda: model.predict_pose_coarse_to_fine(qry[:Q], ref, [rel[2], rel[3]], hier, tposes, k=5,
                                                             keep=keep)
        return lambda: model.predict_pose_refined(qry[:Q], ref, rel[2], refiner, k=5, keep=keep)

    fns = {(c, Q): call(c, Q) for c in cases for Q in args.queries}
    for fn in fns.values():                        # warm every shape (workspace growth, first launches)
        fn()
        fn()
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for Q in args.queries:
            for c in cases:
                samples[(c, Q)].append(timed_ms(fns[(c, Q)], args.iters))

    # top-1 geodesic error on features: query = the engine's template at a seeded off-grid viewpoint
    u = model.u_net
    u.set_metric("l2")
    rf = u.encoder.encode_image(ref)
    qR = viewpoint_rotations(np.random.default_rng(1).standard_normal((args.standin, 3)))
    qf = u.sweep(rf, relative_rotation_6d(qR, ref_R)[None].cuda(), want_emb=True)["emb"]   # [1, n, C, 32, 32]
    qR = torch.from_numpy(qR)
    err = {}
    for c in cases:
        name, keep = c
        if name == "exhaustive":
            R = torch.from_numpy(Rl[keep])[u.sweep(rf, rel[keep], query_feat=qf, want_emb=False,
                                                   k=1)["topi"][0, :, 0].cpu()]
        elif name == "c2f 2->3":
            R = tposes[search(u, rf, qf, [rel[2], rel[3]], hier, keep=keep, k=1)["topi"][0, :, 0].cpu()]
        else:
            seeds = u.sweep(rf, rel[2], query_feat=qf, want_emb=False, k=keep)["topi"]
            out = refine(u, rf, qf, rel[2], seeds, refiner, k=1)
            R = template_rotations(out["D"][0, :, 0], out["seed"][0, :, 0], refiner).cpu()
        e = geodesic_deg(R, qR)
        err[c] = (float(e.median()), float(e.quantile(0.9)))
    torch.cuda.synchronize()

    lines = []
    for Q in args.queries:
        for c in cases:
            name, keep = c
            ms = samples[(c, Q)]
            if name == "exhaustive":
                hyps = len(Rl[keep])
            elif name == "c2f 2->3":
                hyps = hier.sizes[0] + Q * (hier.hypotheses(keep) - hier.sizes[0])
            else:
                hyps = refiner.num_poses + Q * (refiner.hypotheses(keep) - refiner.num_poses)
            lines.append({"case": f"exhaustive level {keep}" if name == "exhaustive" else name,
                          "keep": None if name == "exhaustive" else keep,
                          "steps": args.steps if name == "refine" else None, "Q": Q,
                          "precision": args.precision, "hypotheses": hyps,
                          "ms_per_call": round(statistics.median(ms), 3), "ms_min": round(min(ms), 3),
                          "ms_max": round(max(ms), 3), "top1_err_median_deg": round(err[c][0], 3),
                          "top1_err_p90_deg": round(err[c][1], 3), "standin_queries": args.standin, **info})
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
