"""Time the T-LESS evaluation kernels per frame: render_depth (1 ground-truth + 5 estimated poses) and vsd_errors at
720x540 with the Primesense intrinsics, for B in {1, 16} frames and icospheres of 1.3 k, 20 k and 330 k triangles
plus the 12-triangle box, whose faces are large on screen.  The CPU oracle's time per frame
(oracle/render_oracle.py, torch on the CPU) is printed beside it for scale: it is not pyrender, which cannot run here.

    python tools/vsd_time.py [--reps 5] [--cpu-oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nope_b200.vsd import Mesh, render_depth, vsd_errors   # noqa: E402
from oracle import render_oracle as ro                     # noqa: E402

K = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]])
H, W = 540, 720


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def meshes():
    # icospheres of 20 * 4^s triangles: s = 3, 5, 7 give 1280, 20480 and 327680
    out = {"box (12)": ro.box(60.0, 40.0, 30.0)}
    for s in (3, 5, 7):
        v, f = ro.sphere(40.0, s)
        out[f"sphere ({len(f)})"] = (v, f)
    return out


def time_frames(mesh, B, reps):
    rng = np.random.default_rng(0)
    poses = []
    for b in range(B):
        rot = rng.normal(size=3)
        t = (rng.uniform(-40, 40), rng.uniform(-30, 30), rng.uniform(500, 800))
        poses.append(np.stack([ro.look_pose(*(rot + (0 if p == 0 else rng.normal(0, 0.3, 3))), t=t)
                               for p in range(6)]))
    poses = torch.from_numpy(np.stack(poses)).cuda()
    depth_test = torch.zeros((B, H, W), dtype=torch.float64, device="cuda")
    Kd = torch.from_numpy(np.repeat(K[None], B, axis=0)).cuda()
    r = torch.stack([render_depth(mesh, poses[b], K, (H, W)) for b in range(B)])
    depth_test.copy_(r[:, 0].double())
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_r, t_v = [], []
    for _ in range(reps):
        ev[0].record()
        r = torch.stack([render_depth(mesh, poses[b], K, (H, W)) for b in range(B)])
        ev[1].record()
        vsd_errors(depth_test, r[:, 0], r[:, 1:], Kd)
        ev[2].record()
        torch.cuda.synchronize()
        t_r.append(ev[0].elapsed_time(ev[1]))
        t_v.append(ev[1].elapsed_time(ev[2]))
    return float(np.median(t_r)) / B, float(np.median(t_v)) / B


def time_oracle(v, f):
    """one frame: 6 renders and 5 VSD errors on the CPU oracle"""
    poses = np.stack([ro.look_pose(0.3, 0.2, 0.1 * p, t=(0, 0, 600)) for p in range(6)])
    t0 = time.perf_counter()
    d = ro.render(v, f, poses, K, (H, W)).numpy()
    t1 = time.perf_counter()
    ro.vsd(d[0].astype(np.float64), d[0], d[1:], K)
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-oracle", action="store_true", help="also time the CPU oracle (slow for big meshes)")
    a = ap.parse_args()
    name, pl = card()
    print(f"# {name}, power limit {pl}; 720x540, 1 gt + 5 estimated poses per frame; ms per frame, median of "
          f"{a.reps}")
    rows = []
    for label, (v, f) in meshes().items():
        mesh = Mesh(v, f)
        for B in (1, 16):
            render_depth(mesh, np.eye(4, dtype=np.float32), K, (H, W))       # warm-up
            tr, tv = time_frames(mesh, B, a.reps)
            row = {"mesh": label, "B": B, "render_ms_per_frame": round(tr, 3), "vsd_ms_per_frame": round(tv, 3)}
            if a.cpu_oracle and B == 1 and len(f) <= 2000:
                orr, orv = time_oracle(v, f)
                row.update(cpu_oracle_render_ms=round(orr, 1), cpu_oracle_vsd_ms=round(orv, 1))
            rows.append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps({"card": name, "power_limit": pl, "rows": rows}))


if __name__ == "__main__":
    main()
