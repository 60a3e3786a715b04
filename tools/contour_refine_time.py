"""Time and measure `refine_pose_contour` (DESIGN.md section 20) at 720x540 with the Primesense intrinsics.

Timing: F in {1, 16} frames, P = 5 hypotheses per frame, the default iterations, for the 12-triangle box, a
20 480-triangle icosphere and a 195 840-triangle UV sphere; per call (CUDA events around the Python call, median of
--reps) and per hypothesis.  The split of one call's device time between the rasterizer's kernels ("render": fill,
raster, finish), the distance transform ("sdf": mask_sdf_*) and the fit's own kernels ("fit": init, mask and
silhouette statistics, accumulate, solve, final) comes from torch.profiler in a separate run.  The card's name and
power limit are read in the same run.

With --accuracy it first prints the convergence table: 16 seeded true poses per mesh at 400 - 900 mm, objects inside
the frame, rotations 2.5 - 5 deg off and translations either 5 - 10 mm off ("offset") or from estimate_translation at
the perturbed rotation ("box fit"); the mask is the render at the true pose ("exact") or that render dilated (even
frames) or eroded (odd frames) by one pixel ("+-1 px").  Median and max rotation error (deg) and translation error
(mm) after `iters` updates of the tolerance schedule default_tau(iters, start, end), for several (start, end).

    python tools/contour_refine_time.py [--reps 20] [--accuracy]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from _scenes import K4, angle, scene                                           # noqa: E402
from nope_b200 import contour_refine                                           # noqa: E402
from nope_b200.contour_refine import refine_pose_contour                       # noqa: E402
from nope_b200.translation import estimate_translation                         # noqa: E402
from nope_b200.vsd import Mesh                                                 # noqa: E402
from oracle import render_oracle as ro                                         # noqa: E402
from translation_time import card, timed, uv_sphere                            # noqa: E402

SCHEDULES = [(0.15, 0.02), (0.3, 0.02), (0.15, 0.05), (0.08, 0.02)]
ITERS = [0, 2, 4, 6, 8, 10, 12]


def kernel_split(fn, reps):
    """device time per call (ms) of the rasterizer's kernels (depth_*), the distance transform (mask_sdf_*) and the
    fit's own kernels (contour_*, fit_stats_*), from torch.profiler in a run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    render = sdf = fit = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        if "depth_" in e.key:
            render += us
        elif "mask_sdf_" in e.key:
            sdf += us
        elif "contour_" in e.key or "fit_stats_" in e.key:
            fit += us
    return render / reps / 1e3, sdf / reps / 1e3, fit / reps / 1e3


def _diameter(v):
    v = np.asarray(v, dtype=np.float64)
    return float(max(np.linalg.norm(v - p, axis=1).max() for p in v))


def _detector_masks(M):
    """the masks dilated (even frames) or eroded (odd frames) by one pixel (3 x 3 neighbourhood)"""
    m = M.float()[:, None]
    dil = torch.nn.functional.max_pool2d(m, 3, 1, 1)
    ero = 1 - torch.nn.functional.max_pool2d(1 - m, 3, 1, 1)
    even = (torch.arange(M.shape[0], device=M.device) % 2 == 0)[:, None, None, None]
    return torch.where(even, dil, ero)[:, 0].to(torch.uint8)


def accuracy_table():
    meshes = {"box (12)": ro.box(), "icosphere (320)": ro.sphere(40.0, 2), "soup (64)": ro.soup(64, seed=1)}
    rows = []
    for name, (v, f) in meshes.items():
        mesh = Mesh(v, f)
        R_true, t_true, _, M, R0, t0 = scene(mesh, 100, 16, 1, sensor=False, background=False)
        tb, _ = estimate_translation(mesh, R0, K4, M, diameter=_diameter(v))
        for start, ts in (("offset", t0), ("box fit", tb.cpu().numpy())):
            for mname, masks in (("exact", M), ("+-1 px", _detector_masks(M))):
                for a, b in SCHEDULES:
                    for it in ITERS:
                        R, t, fit = refine_pose_contour(mesh, R0, ts, K4, masks, iters=it,
                                                    tau=contour_refine.default_tau(it, a, b))
                        R, t = R[:, 0].cpu().numpy(), t[:, 0].cpu().numpy()
                        er = np.array([angle(R[i], R_true[i]) for i in range(16)])
                        et = np.linalg.norm(t - t_true, axis=1)
                        iou = fit["iou"][:, 0].cpu().numpy()
                        rows.append({"mesh": name, "start": start, "mask": mname, "tau": [a, b], "iters": it,
                                     "rot_med": float(np.median(er)), "rot_max": float(er.max()),
                                     "t_med": float(np.median(et)), "t_max": float(et.max()),
                                     "iou_min": float(iou.min())})
                        r = rows[-1]
                        print(f"{name:16s} {start:7s} {mname:6s} tau {a:.2f}..{b:.2f} iters {it:2d}: "
                              f"rot deg median {r['rot_med']:.3f} max {r['rot_max']:.3f}; "
                              f"t mm median {r['t_med']:.3f} max {r['t_max']:.3f}; iou min {r['iou_min']:.3f}",
                              flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--accuracy", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contour_refine_time.py needs a CUDA GPU")
    name, pl = card()
    iters = contour_refine.DEFAULT_ITERS
    print(f"# {name}, power limit {pl}; 720x540, P = 5, iters {iters}; CUDA events, median of {a.reps}")
    out = {"card": name, "power_limit": pl}
    if a.accuracy:
        out["accuracy"] = accuracy_table()
    meshes = {"box (12)": ro.box(), "icosphere (20480)": ro.sphere(40.0, 5), "uv sphere (195840)": uv_sphere()}
    rows, P = [], 5
    for mname, (v, f) in meshes.items():
        mesh = Mesh(v, f)
        for F in (1, 16):
            _, _, _, M, R0, t0 = scene(mesh, 1, F, P, sensor=False, background=False)
            Rd, td = torch.from_numpy(R0).cuda(), torch.from_numpy(t0).cuda()
            call = lambda: refine_pose_contour(mesh, Rd, td, K4, M, iters=iters)   # noqa: E731
            ms = timed(call, a.reps)
            render, sdf, fit = kernel_split(call, a.reps)
            row = {"mesh": mname, "F": F, "P": P, "iters": iters, "ms": ms, "us_per_hyp": 1e3 * ms / (F * P),
                   "ms_render_kernels": render, "ms_sdf_kernels": sdf, "ms_fit_kernels": fit}
            rows.append(row)
            print(f"{mname:20s} F {F:2d}: {ms:.3f} ms ({row['us_per_hyp']:.1f} us / hypothesis); kernels: render "
                  f"{render:.3f} ms, sdf {sdf:.3f} ms, fit {fit:.3f} ms", flush=True)
    out["rows"] = rows
    print(json.dumps(out))


if __name__ == "__main__":
    main()
