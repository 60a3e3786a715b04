"""Time predict_pose for one reference, N poses and Q query images, two ways, in ONE process:
  (a) multi-query: predict_pose(query [Q, 3, 256, 256], reference [1, ...], all_relativeR [1, N, 6]) -- one sweep;
  (b) repeated reference: reference and pose grid repeated Q times, B = Q -- Q sweeps of identical templates.
    python tools/multi_query_time.py --poses 642 --queries 1 4 16 64 --reps 5 --out /tmp/multi_query.json
Device events around whole calls (encoder + sweep + scoring + top-k), warm-up of every shape, the two ways
alternated inside each repetition; ms is the median over repetitions with the min / max beside it.  A separate
torch.profiler run then reads the fused score kernel (final_conv_score_kernel) and the top-k kernel alone.
Prints the card name and power limit with the numbers.  A development aid, not the bench."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200 import synth_weights as weights
from nope_b200.model import build_model
from nope_b200.poses import synthetic_pose_batch


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:                        # the numbers are still printed, labelled as unknown card
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc.__class__.__name__})"}


def timed_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn, names, iters=3):
    """device time per call of the kernels whose names contain one of `names` (torch.profiler, own run)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                us = getattr(ev, "device_time_total", None)
                if us is None:
                    us = ev.cuda_time_total
                out[n] += us / 1e3 / iters
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=642)
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--reps", type=int, default=5, help="alternating repetitions of every (Q, way) pair")
    ap.add_argument("--iters", type=int, default=2, help="calls per timed window")
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_query_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0", precision=args.precision).load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    N = args.poses
    poses, _ = synthetic_pose_batch(N, 1)
    poses = poses.cuda()
    g = torch.Generator().manual_seed(0)
    ref = torch.rand(1, 3, 256, 256, generator=g).cuda()
    qmax = max(args.queries)
    qry = torch.rand(qmax, 3, 256, 256, generator=g).cuda()

    def way_a(Q):
        return lambda: model.predict_pose(qry[:Q], ref, poses, None, k=5)

    def way_b(Q):
        refs, grid = ref.expand(Q, -1, -1, -1).contiguous(), poses.expand(Q, -1, -1).contiguous()
        return lambda: model.predict_pose(qry[:Q], refs, grid, None, k=5)

    fns = {(Q, w): (way_a(Q) if w == "a" else way_b(Q)) for Q in args.queries for w in ("a", "b")}
    for fn in fns.values():                        # warm every shape (workspace growth, first launches)
        fn()
        fn()
    # the two ways give the same ranking
    for Q in args.queries:
        _, ia, sa = fns[(Q, "a")]()
        _, ib, sb = fns[(Q, "b")]()
        assert torch.equal(ia, ib), Q
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for Q in args.queries:
            for w in ("a", "b"):
                samples[(Q, w)].append(timed_ms(fns[(Q, w)], args.iters))
    lines = []
    for Q in args.queries:
        for w in ("a", "b"):
            ms = samples[(Q, w)]
            med = statistics.median(ms)
            lines.append({"Q": Q, "way": "multi_query" if w == "a" else "repeat_reference", "poses": N,
                          "precision": args.precision, "ms_per_call": round(med, 3),
                          "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3),
                          "queries_per_s": round(Q / (med * 1e-3), 1), **info})
    # what grows with Q on the multi-query path besides the scoring: encoding the Q query images
    enc = model.u_net.encoder
    for Q in args.queries:
        ms = [timed_ms(lambda: enc.encode_image(torch.cat([qry[:Q], ref])), args.iters) for _ in range(args.reps)]
        lines.append({"Q": Q, "way": "encoder_only", "images": Q + 1, "ms_per_call": round(statistics.median(ms), 3),
                      "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), **info})
    # kernel times, profiler on, separate run
    for Q in args.queries:
        k = kernel_ms(fns[(Q, "a")], ["final_conv_score_kernel", "sim_topk_kernel"])
        lines.append({"Q": Q, "way": "multi_query", "profile": "torch.profiler, own run",
                      "final_conv_score_kernel_ms": round(k["final_conv_score_kernel"], 4),
                      "sim_topk_kernel_ms": round(k["sim_topk_kernel"], 4), **info})
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
