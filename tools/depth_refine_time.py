"""Time and measure `refine_pose_depth` (DESIGN.md section 19) at 720x540 with the Primesense intrinsics.

Timing: F in {1, 16} frames, P = 5 hypotheses per frame, the default iterations, for the 12-triangle box, a
20 480-triangle icosphere and a 195 840-triangle UV sphere; per call (CUDA events around the Python call, median of
--reps) and per hypothesis.  The split of one call's device time between the rasterizer's kernels ("render": fill,
raster, finish) and the refinement's own kernels ("icp": init, valid count, accumulate, solve, final) comes from
torch.profiler in a separate run.  The card's name and power limit are read in the same run.

With --accuracy it first prints the convergence table: 16 seeded true poses per mesh at 400 - 900 mm, objects inside
the frame, starts 2.5 - 5 deg and 5 - 10 mm off, the mask, and a background plane 40 mm behind the object; the sensor
depth is the render at the true pose, exact ("clean") or with 0.5 mm noise, 2 % holes and 0.1 mm quantisation
("noisy").  Median and max rotation error (deg) and translation error (mm) after `iters` updates of the tolerance
schedule TAU_START d ... TAU_END d, for several schedules.

    python tools/depth_refine_time.py [--reps 20] [--accuracy]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from _scenes import K4, angle, scene                                           # noqa: E402
from nope_b200 import depth_refine                                             # noqa: E402
from nope_b200.depth_refine import refine_pose_depth                           # noqa: E402
from nope_b200.vsd import Mesh                                                 # noqa: E402
from oracle import render_oracle as ro                                         # noqa: E402
from translation_time import card, timed, uv_sphere                            # noqa: E402

SCHEDULES = [(0.25, 0.02), (0.5, 0.02), (0.5, 0.05), (1.0, 0.02)]
ITERS = [0, 1, 2, 3, 4, 6, 8, 10]


def kernel_split(fn, reps):
    """device time per call (ms) of the rasterizer's kernels (depth_*) and of the refinement's kernels (icp_*), from
    torch.profiler in a run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    render = icp = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        if "depth_" in e.key:
            render += us
        elif "icp_" in e.key:
            icp += us
    return render / reps / 1e3, icp / reps / 1e3


def accuracy_table():
    meshes = {"box (12)": ro.box(), "icosphere (320)": ro.sphere(40.0, 2), "soup (64)": ro.soup(64, seed=1)}
    rows = []
    default = (depth_refine.TAU_START, depth_refine.TAU_END)
    try:
        for name, (v, f) in meshes.items():
            mesh = Mesh(v, f)
            for noisy in (False, True):
                R_true, t_true, S, M, R0, t0 = scene(mesh, 100, 16, 1, sensor=noisy)
                for a, b in SCHEDULES:
                    depth_refine.TAU_START, depth_refine.TAU_END = a, b
                    for it in ITERS:
                        R, t, fit = refine_pose_depth(mesh, R0, t0, K4, S, masks=M, iters=it)
                        R, t = R[:, 0].cpu().numpy(), t[:, 0].cpu().numpy()
                        er = np.array([angle(R[i], R_true[i]) for i in range(16)])
                        et = np.linalg.norm(t - t_true, axis=1)
                        sc = fit["score"][:, 0].cpu().numpy()
                        rows.append({"mesh": name, "noise": noisy, "tau": [a, b], "iters": it,
                                     "rot_med": float(np.median(er)), "rot_max": float(er.max()),
                                     "t_med": float(np.median(et)), "t_max": float(et.max()),
                                     "score_min": float(sc.min())})
                        r = rows[-1]
                        print(f"{name:16s} {'noisy' if noisy else 'clean'} tau {a:.2f}..{b:.2f} d iters {it:2d}: "
                              f"rot deg median {r['rot_med']:.4f} max {r['rot_max']:.4f}; "
                              f"t mm median {r['t_med']:.4f} max {r['t_max']:.4f}; score min {r['score_min']:.3f}",
                              flush=True)
    finally:
        depth_refine.TAU_START, depth_refine.TAU_END = default
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--accuracy", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_refine_time.py needs a CUDA GPU")
    name, pl = card()
    iters = depth_refine.DEFAULT_ITERS
    print(f"# {name}, power limit {pl}; 720x540, P = 5, iters {iters}; CUDA events, median of {a.reps}")
    out = {"card": name, "power_limit": pl}
    if a.accuracy:
        out["accuracy"] = accuracy_table()
    meshes = {"box (12)": ro.box(), "icosphere (20480)": ro.sphere(40.0, 5), "uv sphere (195840)": uv_sphere()}
    rows, P = [], 5
    for mname, (v, f) in meshes.items():
        mesh = Mesh(v, f)
        for F in (1, 16):
            _, _, S, M, R0, t0 = scene(mesh, 1, F, P)
            Rd, td = torch.from_numpy(R0).cuda(), torch.from_numpy(t0).cuda()
            call = lambda: refine_pose_depth(mesh, Rd, td, K4, S, masks=M, iters=iters)   # noqa: E731
            ms = timed(call, a.reps)
            render, icp = kernel_split(call, a.reps)
            row = {"mesh": mname, "F": F, "P": P, "iters": iters, "ms": ms, "us_per_hyp": 1e3 * ms / (F * P),
                   "ms_render_kernels": render, "ms_icp_kernels": icp}
            rows.append(row)
            print(f"{mname:20s} F {F:2d}: {ms:.3f} ms ({row['us_per_hyp']:.1f} us / hypothesis); kernels: render "
                  f"{render:.3f} ms, icp {icp:.3f} ms", flush=True)
    out["rows"] = rows
    print(json.dumps(out))


if __name__ == "__main__":
    main()
