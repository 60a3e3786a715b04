"""Time the resident sweep (latents + poses in HBM, CUDA events on the current stream) for one or
several engine precisions in ONE process, e.g.
    python tools/time_sweep.py fp16 parity fp16_w2 --poses 642 --queries 1
Prints one JSON line per precision (hyp/s, ms, parity vs the first one's scores) -- a development aid,
not the bench."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200 import synth_weights as weights
from nope_b200.model import build_model
from nope_b200.poses import synthetic_pose_batch

ap = argparse.ArgumentParser()
ap.add_argument("precisions", nargs="+")
ap.add_argument("--poses", type=int, default=642)
ap.add_argument("--queries", type=int, default=1)
ap.add_argument("--chunk", type=int, default=642)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--profile", action="store_true", help="per-launch conv timing (CUDA events)")
args = ap.parse_args()

sd = weights.make_full_state_dict(seed=0)
poses, _ = synthetic_pose_batch(args.poses, args.queries)
g = torch.Generator().manual_seed(0)
rf = (torch.randn(args.queries, 8, 32, 32, generator=g) * 1.5).cuda()
qf = (torch.randn(args.queries, 8, 32, 32, generator=g) * 1.5).cuda()
poses = poses.cuda()
base = None
for prec in args.precisions:
    model = build_model(device="cuda:0", chunk=args.chunk, precision=prec)
    model.load_state_dict(sd)
    u = model.u_net
    run = lambda: u.sweep(rf, poses, query_feat=qf, want_emb=False, k=5)
    for _ in range(3):
        out = run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    line = {"precision": prec, "ms": ms, "hyp_per_s": args.queries * args.poses / (ms * 1e-3),
            "launches": u.last_launch_count, "top5": out["topi"][0].tolist(),
            "sim_crc": __import__("zlib").crc32(out["sim"].float().cpu().numpy().tobytes())}
    if base is None:
        base = out["sim"].clone()
    else:
        d = (out["sim"] - base).abs().max() / base.abs().max()
        line["sim_max_rel_vs_first"] = float(d)
    if args.profile:
        u.profile(True)
        run()
        p = u.profile_read()
        u.profile(False)
        line.update(conv_ms=p["conv_ms"], conv_exec_tflops=p["conv_flops"] / (p["conv_ms"] * 1e-3) / 1e12,
                    conv_alg_tflops=p["conv_alg_flops"] / (p["conv_ms"] * 1e-3) / 1e12, conv_launches=p["conv_launches"])
    print(json.dumps(line), flush=True)
    del model, u
    torch.cuda.empty_cache()
