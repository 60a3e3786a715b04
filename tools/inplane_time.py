"""Time the in-plane rotation search against predict_pose for one reference, N poses and Q query images, in ONE
process:
  predict_pose           one encoder call (Q + 1 images), one sweep, top-k;
  predict_pose_inplane   A angles: the reference encoded, the Q * A rotated copies encoded 32 at a time through the
                         staging buffer, one sweep with Q * A query rows, the joint top-k.
Each case is also split into its encoder part (encode_image / encode_image_inplane alone) and the rest
(sweep + scoring + top-k on precomputed features).
    python tools/inplane_time.py --angles 1 12 36 72 --queries 1 16 --reps 5 --out /tmp/inplane.json
Device events around whole calls, warm-up of every shape, the cases alternated inside each repetition; ms is the
median over repetitions with the min / max beside it.  Prints the card name and power limit with the numbers.
Seeded weights: the times do not depend on them, and nothing here measures how well a roll is recovered.  A
development aid, not the bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200 import synth_weights as weights
from nope_b200.model import build_model, topk
from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=642)
    ap.add_argument("--angles", type=int, nargs="+", default=[1, 12, 36, 72])
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--reps", type=int, default=5, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=2, help="calls per timed window")
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inplane_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0", precision=args.precision).load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    u, enc = model.u_net, model.u_net.encoder
    N = args.poses
    rel = synthetic_pose_batch(N, 1)[0].cuda()
    tp = torch.from_numpy(icosphere_object_rotations(2)).cuda() if N == 642 else None
    g = torch.Generator().manual_seed(0)
    ref = torch.rand(1, 3, 256, 256, generator=g).cuda() * 2 - 1
    qry = torch.rand(max(args.queries), 3, 256, 256, generator=g).cuda() * 2 - 1
    u.set_metric("l2")
    ref_feat = enc.encode_image(ref)
    # (name, A): A = 0 is predict_pose
    cases = [("predict_pose", 0)] + [("predict_pose_inplane", A) for A in args.angles]

    def whole(case, Q):
        name, A = case
        if A == 0:
            return lambda: model.predict_pose(qry[:Q], ref, rel, tp, k=5)
        return lambda: model.predict_pose_inplane(qry[:Q], ref, rel, tp, k=5, angles=A)

    def encoder_part(case, Q):
        _, A = case
        if A == 0:
            return lambda: enc.encode_image(torch.cat([qry[:Q], ref]))
        return lambda: (enc.encode_image(ref), enc.encode_image_inplane(qry[:Q], A))

    feats = {}

    def sweep_part(case, Q):
        _, A = case
        if A == 0:
            qf = enc.encode_image(qry[:Q])[None]
            return lambda: u.sweep(ref_feat, rel, query_feat=qf, want_emb=False, k=5)
        qf = feats.setdefault((A, Q), enc.encode_image_inplane(qry[:Q], A).view(1, Q * A, -1, 32, 32))

        def run():
            sim = u.sweep(ref_feat, rel, query_feat=qf, want_emb=False, want_sim=True, k=0)["sim"]
            return topk(sim.view(Q, A * N), 5)
        return run

    parts = {"whole": whole, "encoder": encoder_part, "sweep": sweep_part}
    fns = {(c, Q, p): mk(c, Q) for c in cases for Q in args.queries for p, mk in parts.items()}
    for fn in fns.values():                        # warm every shape (workspace growth, staging buffer, first launches)
        fn()
        fn()
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for key, fn in fns.items():
            samples[key].append(timed_ms(fn, args.iters))

    lines = []
    for Q in args.queries:
        base = statistics.median(samples[(cases[0], Q, "whole")])
        for c in cases:
            name, A = c
            row = {"case": name, "angles": A or None, "Q": Q, "poses": N, "precision": args.precision,
                   "encoded_images": Q + 1 if A == 0 else Q * A + 1, "query_rows": Q * max(A, 1)}
            for p in parts:
                ms = samples[(c, Q, p)]
                row[f"{p}_ms"] = round(statistics.median(ms), 3)
                row[f"{p}_ms_min"] = round(min(ms), 3)
                row[f"{p}_ms_max"] = round(max(ms), 3)
            row["extra_ms_over_predict_pose"] = round(row["whole_ms"] - base, 3)
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
