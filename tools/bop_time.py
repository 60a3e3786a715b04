"""Time the BOP 2019 error kernels: pose_errors (MSSD + MSPD) over S in {1, 315, 630} symmetry transforms x V in
{2 k, 20 k, 200 k} model points x B*k in {5, 80} estimates, and the VSD of 1 ground-truth + 5 estimated poses per frame
at 720x540 as ten single-tau vsd_errors calls against one ten-tau call, for B in {1, 16} frames.  The card's name and
power limit are read in the same run.

    python tools/bop_time.py [--reps 5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nope_b200 import bop                                              # noqa: E402
from nope_b200.vsd import Mesh, render_depth, vsd_errors               # noqa: E402
from oracle import render_oracle as ro                                 # noqa: E402
from tools.vsd_time import H, K, W, card                               # noqa: E402

CYL = {"symmetries_discrete": [np.diag([1.0, -1.0, -1.0, 1.0])],
       "symmetries_continuous": [{"axis": np.array([0.0, 0.0, 1.0]), "offset": np.zeros(3)}]}


def _events(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    out = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(out))


def time_pose_errors(reps):
    syms = {1: np.eye(3, 4)[None], 315: bop.symmetry_transformations({"symmetries_continuous":
                                                                        CYL["symmetries_continuous"]}),
            630: bop.symmetry_transformations(CYL)}
    rng = np.random.default_rng(0)
    K4 = torch.tensor([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=torch.float64)
    rows = []
    for V in (2000, 20000, 200000):
        pts = torch.from_numpy(rng.normal(0, 40, (V, 3)).astype(np.float32)).cuda()
        for n in (5, 80):
            F, P = (1, 5) if n == 5 else (16, 5)
            poses = [ro.look_pose(*rng.normal(size=3), t=(0, 0, 700)).astype(np.float64) for _ in range(F * (P + 1))]
            poses = torch.from_numpy(np.stack(poses)).cuda()
            R_gt, t_gt = poses[:F, :3, :3], poses[:F, :3, 3]
            R_est, t_est = poses[F:, :3, :3].reshape(F, P, 3, 3), poses[F:, :3, 3].reshape(F, P, 3)
            for S, sy in syms.items():
                sd = torch.from_numpy(sy).cuda()
                ms = _events(lambda: bop.pose_errors(pts, R_est, t_est, R_gt, t_gt, K4, sd), reps)
                row = {"what": "pose_errors", "S": S, "V": V, "estimates": F * P, "ms": round(ms, 4),
                       "G_point_syms_per_s": round(S * V * F * P / ms / 1e6, 2)}
                rows.append(row)
                print(json.dumps(row), flush=True)
    return rows


def time_vsd(reps):
    v, f = ro.sphere(40.0, 5)
    mesh = Mesh(v, f)
    rng = np.random.default_rng(1)
    rows = []
    for B in (1, 16):
        poses = []
        for _ in range(B):
            rot, t = rng.normal(size=3), (rng.uniform(-40, 40), rng.uniform(-30, 30), rng.uniform(500, 800))
            poses.append(np.stack([ro.look_pose(*(rot + (0 if p == 0 else rng.normal(0, 0.3, 3))), t=t)
                                   for p in range(6)]))
        r = torch.stack([render_depth(mesh, torch.from_numpy(p).cuda(), K, (H, W)) for p in poses])
        dt, dg, de = r[:, 0].double(), r[:, 0].contiguous(), r[:, 1:].contiguous()
        Kh = np.repeat(np.array([[K[0, 0], K[1, 1], K[0, 2], K[1, 2]]]), B, axis=0)
        Kd = torch.from_numpy(Kh).cuda()
        taus = bop.VSD_TAUS * 80.0
        single = _events(lambda: [vsd_errors(dt, dg, de, Kd, tau=float(t)) for t in taus], reps)
        multi = _events(lambda: vsd_errors(dt, dg, de, Kh, tau=taus), reps)
        row = {"what": "vsd", "B": B, "estimates_per_frame": 5, "ten_single_tau_ms": round(single, 4),
               "one_ten_tau_ms": round(multi, 4), "speedup": round(single / multi, 2)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, pl = card()
    print(f"# {name}, power limit {pl}; CUDA events, median of {a.reps}")
    rows = time_pose_errors(a.reps) + time_vsd(a.reps)
    print(json.dumps({"card": name, "power_limit": pl, "rows": rows}))


if __name__ == "__main__":
    main()
