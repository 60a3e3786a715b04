"""Time the coarse-to-fine pose search against the exhaustive sweep over the synthetic level-3 grid (2562 poses),
for one reference and Q query images, in ONE process:
  exhaustive   predict_pose over all 2562 poses;
  2->3         predict_pose_coarse_to_fine over levels 2, 3 (642 -> 2562) with keep in --keeps;
  1->2->3      levels 1, 2, 3 (162 -> 642 -> 2562) with keep 8.
    python tools/coarse_to_fine_time.py --queries 1 16 --reps 5 --out /tmp/c2f.json
Device events around whole calls (encoder + every stage), warm-up of every shape, the cases alternated inside each
repetition; ms is the median over repetitions with the min / max beside it.  `hypotheses` is what one call sweeps.

Top-1 agreement with the exhaustive search is measured on features, not images: --agree seeded off-grid query
rotations, each query feature the engine's own template at that rotation (a stand-in for a real query: no trained
checkpoint exists, so the figure says how often the cells hold the best pose of a smooth seeded-weight score
landscape, nothing about trained weights).  Prints the card name and power limit with the numbers.  A development
aid, not the bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200 import synth_weights as weights
from nope_b200.hierarchy import PoseHierarchy, search
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def random_rotations(n, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((n, 4), generator=g, dtype=torch.float64)
    w, x, y, z = (q / q.norm(dim=1, keepdim=True)).unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
                       dim=1).reshape(n, 3, 3).numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--keeps", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--reps", type=int, default=5, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=3, help="calls per timed window")
    ap.add_argument("--agree", type=int, default=64, help="seeded off-grid queries for the top-1 agreement")
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("coarse_to_fine_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0", precision=args.precision).load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    Rl = {l: icosphere_object_rotations(l) for l in (1, 2, 3)}
    ref_R = Rl[3][7]
    rel = {l: relative_rotation_6d(Rl[l], ref_R)[None].cuda() for l in Rl}
    tposes = torch.from_numpy(Rl[3])
    hier = {"2->3": PoseHierarchy([Rl[2], Rl[3]]), "1->2->3": PoseHierarchy([Rl[1], Rl[2], Rl[3]])}
    cases = [("exhaustive", None, None)] + [("2->3", k, (2, 3)) for k in args.keeps] + [("1->2->3", 8, (1, 2, 3))]

    g = torch.Generator().manual_seed(0)
    ref = torch.rand(1, 3, 256, 256, generator=g).cuda()
    qry = torch.rand(max(args.queries), 3, 256, 256, generator=g).cuda()

    def call(case, Q):
        name, keep, levels = case
        if name == "exhaustive":
            return lambda: model.predict_pose(qry[:Q], ref, rel[3], tposes, k=5)
        return lambda: model.predict_pose_coarse_to_fine(qry[:Q], ref, [rel[l] for l in levels], hier[name],
                                                         tposes, k=5, keep=keep)

    fns = {(c, Q): call(c, Q) for c in cases for Q in args.queries}
    for fn in fns.values():                        # warm every shape (workspace growth, first launches)
        fn()
        fn()
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for Q in args.queries:
            for c in cases:
                samples[(c, Q)].append(timed_ms(fns[(c, Q)], args.iters))

    # top-1 agreement on features: query = the engine's template at a seeded off-grid rotation
    u = model.u_net
    model.u_net.set_metric("l2")
    rf = model.u_net.encoder.encode_image(ref)
    qR = random_rotations(args.agree, seed=1)
    qrel = relative_rotation_6d(qR, ref_R)[None].cuda()
    qf = u.sweep(rf, qrel, want_emb=True)["emb"]                          # [1, n, C, 32, 32]
    ex_top = u.sweep(rf, rel[3], query_feat=qf, want_emb=False, k=1)["topi"][0, :, 0]
    agree = {}
    for c in cases[1:]:
        name, keep, levels = c
        out = search(u, rf, qf, [rel[l] for l in levels], hier[name], keep=keep, k=1)
        agree[c] = float((out["topi"][0, :, 0] == ex_top).float().mean())
    torch.cuda.synchronize()

    lines = []
    for Q in args.queries:
        for c in cases:
            name, keep, levels = c
            ms = samples[(c, Q)]
            hyps = 2562 if name == "exhaustive" else \
                hier[name].sizes[0] + Q * (hier[name].hypotheses(keep) - hier[name].sizes[0])
            lines.append({"case": name, "keep": keep, "Q": Q, "poses": 2562, "precision": args.precision,
                          "hypotheses": hyps, "ms_per_call": round(statistics.median(ms), 3),
                          "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3),
                          "top1_agreement": 1.0 if name == "exhaustive" else agree[c],
                          "agreement_queries": args.agree, **info})
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
