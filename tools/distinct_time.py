"""Time the distinct top-k (nope_distinct_topk, DESIGN.md section 21) beside the sweep that produces its rows, in ONE
process: for one reference and Q queries (B * Q rows), N poses,
  predict_pose            N = 642 (level 2) or 2562 (level 3): its similarity [Q, N];
  predict_pose_inplane    A = 36 over 2562 poses: its similarity flattened to [Q, 36 * 2562];
then distinct_topk of those rows with k = 5 and k = 64 at theta = 20 degrees, for three symmetry groups: none,
a 4-fold discrete group, and a continuous axis with a 2-fold flip (2 discrete rotations).
    python tools/distinct_time.py --queries 1 16 --out /tmp/distinct.json
CUDA events around whole calls after a warm-up of every shape; the selection is the median of --reps calls, the
sweep the median of --sweep-reps.  Prints the card name and power limit with the numbers.  Seeded weights: the
times do not depend on them.  A development aid, not the bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import synth_weights as weights
from nope_b200.distinct import distinct_topk
from nope_b200.inplane import compose
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def _entry(disc, axis=None):
    mats = []
    for R in disc:
        m = np.eye(4)
        m[:3, :3] = R
        mats.append(m)
    return {"symmetries_discrete": mats,
            "symmetries_continuous": [] if axis is None else [{"axis": np.asarray(axis, float)}]}


QUARTER_Z = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
GROUPS = {"none": None,
          "four": _entry([np.linalg.matrix_power(QUARTER_Z, i) for i in (1, 2, 3)]),
          "axis+2": _entry([np.diag([1.0, -1.0, -1.0])], axis=[0.0, 0.0, 1.0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--reps", type=int, default=20, help="timed selection calls (median)")
    ap.add_argument("--sweep-reps", type=int, default=5, help="timed sweeps (median)")
    ap.add_argument("--theta", type=float, default=20.0)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("distinct_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0").load_state_dict(weights.make_full_state_dict(seed=0)).eval()
    g = torch.Generator().manual_seed(0)
    ref = torch.rand(1, 3, 256, 256, generator=g).cuda() * 2 - 1
    qry = torch.rand(max(args.queries), 3, 256, 256, generator=g).cuda() * 2 - 1
    lines = []
    for level, A in ((2, 1), (3, 1), (3, 36)):
        R = torch.from_numpy(icosphere_object_rotations(level)).cuda()
        N = R.shape[0]
        rel = synthetic_pose_batch(N, 1)[0].cuda()
        if A == 1:
            rot = R[None]
        else:
            a, n = torch.arange(A).repeat_interleave(N).cuda(), torch.arange(N).repeat(A).cuda()
            rot = compose(R, n, a, A)[None]
        for Q in args.queries:
            q = qry[:Q][None]                                                       # [1, Q, 3, H, W]
            if A == 1:
                sweep = lambda: model.predict_pose(q, ref, rel, k=5)[2]             # noqa: E731
            else:
                sweep = lambda: model.predict_pose_inplane(q, ref, rel, k=5, angles=A)[3]   # noqa: E731
            sim = sweep().reshape(Q, -1)
            sweep_ms = statistics.median(timed_ms(sweep, 1) for _ in range(args.sweep_reps))
            for gname, sym in GROUPS.items():
                for k in (5, 64):
                    call = lambda: distinct_topk(sim, rot, k, args.theta, sym)      # noqa: E731
                    call()
                    ms = [timed_ms(call, 1) for _ in range(args.reps)]
                    line = {"rows": Q, "N": sim.shape[1], "angles": A, "group": gname, "k": k, "theta": args.theta,
                            "distinct_ms": round(statistics.median(ms), 4), "min_ms": round(min(ms), 4),
                            "max_ms": round(max(ms), 4), "sweep_ms": round(sweep_ms, 3),
                            "share_of_sweep": round(statistics.median(ms) / sweep_ms, 5), **info}
                    print(json.dumps(line), flush=True)
                    lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
