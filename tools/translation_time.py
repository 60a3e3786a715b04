"""Time `estimate_translation` (DESIGN.md section 18) at 720x540 with the Primesense intrinsics: F in {1, 16} frames,
P = 5 rotation hypotheses per frame, iters in {0, 4}, for the 12-triangle box, a 20 480-triangle icosphere and a
195 840-triangle UV sphere.  Per call (CUDA events around the Python call) and per hypothesis; the split of one
iters = 4 call's device time between the rasterizer's kernels ("render": fill, raster, finish) and the fit's own
kernels ("stats + update") comes from torch.profiler in a separate run.  The numpy / torch-CPU oracle
(tests/translation_oracle.py) for one
hypothesis of the box is printed for scale.  CUDA events, median of --reps runs; the card's name and power limit
are read in the same run.

With --accuracy it also prints the convergence table: 32 seeded true poses per mesh at 400 - 1200 mm, objects inside
the frame, masks rendered at the true pose, the fit from `initial_translation` with the true rotation after 0 ... 6
updates: |dz| in units of z / sqrt(w h) (one pixel of box size) and the origin's reprojection error in px.

    python tools/translation_time.py [--reps 20] [--accuracy] [--cpu-oracle]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from nope_b200.translation import estimate_translation, initial_translation   # noqa: E402
from nope_b200.vsd import Mesh, render_depth                                  # noqa: E402
from oracle import render_oracle as ro                                        # noqa: E402

K4 = np.array([1075.65091572, 1073.90347929, 360.0, 270.0])
H, W = 540, 720


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def uv_sphere(radius=40.0, n_lat=256, n_lon=384):
    """closed UV sphere: 2 n_lon (n_lat - 1) triangles (195 840 at the defaults)"""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    v = [[0, 0, radius]] + [[radius * np.sin(a) * np.cos(b), radius * np.sin(a) * np.sin(b), radius * np.cos(a)]
                            for a in th for b in ph] + [[0, 0, -radius]]
    ring = lambda i, j: 1 + i * n_lon + j % n_lon                   # noqa: E731
    f = [[0, ring(0, j), ring(0, j + 1)] for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    last = len(v) - 1
    f += [[last, ring(n_lat - 2, j + 1), ring(n_lat - 2, j)] for j in range(n_lon)]
    return np.array(v, dtype=np.float32), np.array(f, dtype=np.int32)


def diameter(v):
    v = v.astype(np.float64)
    c = v.mean(0)
    return 2.0 * float(np.linalg.norm(v - c, axis=1).max())         # a bound; only the start uses it


def pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T.astype(np.float32)


def rot(rng):
    return ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)


def box_stats(m):
    rows, cols = np.nonzero(m.any(1))[0], np.nonzero(m.any(0))[0]
    return (rows[0], rows[-1], cols[0], cols[-1]) if len(rows) else None


def scene(mesh, seed, F, P):
    rng = np.random.default_rng(seed)
    Rt, tt, masks = [], [], []
    while len(Rt) < F:
        R = rot(rng)
        z = rng.uniform(400, 1200)
        t = np.array([rng.uniform(-0.2, 0.2) * z, rng.uniform(-0.2, 0.2) * z, z])
        m = render_depth(mesh, torch.from_numpy(pose(R, t)), K4, (H, W))[0] > 0
        b = box_stats(m.cpu().numpy())
        if b is None or b[0] == 0 or b[2] == 0 or b[1] == H - 1 or b[3] == W - 1:
            continue
        Rt.append(R), tt.append(t), masks.append(m.to(torch.uint8))
    R = np.stack([np.stack([Rt[f]] + [rot(rng) for _ in range(P - 1)]) for f in range(F)])
    return np.stack(Rt), np.stack(tt), torch.stack(masks), R


def timed(fn, reps):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernel_split(fn, reps):
    """device time per call (ms) of the rasterizer's kernels (depth_*) and of the fit's own kernels (fit_*), from
    torch.profiler in a run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    render = fit = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        if "depth_" in e.key:
            render += us
        elif "fit_" in e.key:
            fit += us
    return render / reps / 1e3, fit / reps / 1e3


def accuracy_table():
    meshes = {"box (12)": ro.box(), "icosphere (320)": ro.sphere(40.0, 2), "soup (64)": ro.soup(64, seed=1)}
    rows = []
    for name, (v, f) in meshes.items():
        mesh = Mesh(v, f)
        d = float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))
        R, t_true, masks, _ = scene(mesh, 100, 32, 1)
        mh = masks.cpu().numpy()
        px = np.array([math.sqrt((b[3] - b[2] + 1) * (b[1] - b[0] + 1)) for b in map(box_stats, mh)])
        ut = K4[:2] * t_true[:, :2] / t_true[:, 2:] + K4[2:]
        for it in range(7):
            t, iou = estimate_translation(mesh, R, K4, masks, diameter=d, iters=it)
            t, iou = t[:, 0].cpu().numpy(), iou[:, 0].cpu().numpy()
            dz = np.abs(t[:, 2] - t_true[:, 2]) / (t_true[:, 2] / px)
            rp = np.hypot(*(K4[:2] * t[:, :2] / t[:, 2:] + K4[2:] - ut).T)
            rows.append({"mesh": name, "iters": it, "dz_med": float(np.median(dz)), "dz_max": float(dz.max()),
                         "reproj_med": float(np.median(rp)), "reproj_max": float(rp.max()),
                         "iou_med": float(np.median(iou)), "iou_min": float(iou.min())})
            r = rows[-1]
            print(f"{name:16s} iters {it}: |dz| / (z / sqrt(wh)) median {r['dz_med']:.3f} max {r['dz_max']:.3f}; "
                  f"reprojection px median {r['reproj_med']:.3f} max {r['reproj_max']:.3f}; "
                  f"IoU median {r['iou_med']:.4f} min {r['iou_min']:.4f}", flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--accuracy", action="store_true")
    ap.add_argument("--cpu-oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("translation_time.py needs a CUDA GPU")
    name, pl = card()
    print(f"# {name}, power limit {pl}; 720x540, P = 5; CUDA events, median of {a.reps}")
    out = {"card": name, "power_limit": pl}
    if a.accuracy:
        out["accuracy"] = accuracy_table()
    meshes = {"box (12)": ro.box(), "icosphere (20480)": ro.sphere(40.0, 5), "uv sphere (195840)": uv_sphere()}
    rows, P = [], 5
    for mname, (v, f) in meshes.items():
        mesh = Mesh(v, f)
        d = diameter(v)
        for F in (1, 16):
            _, _, masks, R = scene(mesh, 1, F, P)
            Rd = torch.from_numpy(R).cuda()
            t0 = initial_translation(masks, K4, d)
            t = {it: timed(lambda: estimate_translation(mesh, Rd, K4, masks, t_init=t0, iters=it), a.reps)
                 for it in (0, 4)}
            render, fit = kernel_split(lambda: estimate_translation(mesh, Rd, K4, masks, t_init=t0, iters=4), a.reps)
            row = {"mesh": mname, "F": F, "P": P, "ms_iters0": t[0], "ms_iters4": t[4],
                   "us_per_hyp_iters4": 1e3 * t[4] / (F * P), "ms_render_kernels_iters4": render,
                   "ms_fit_kernels_iters4": fit}
            rows.append(row)
            print(f"{mname:20s} F {F:2d}: iters 0 {t[0]:.3f} ms, iters 4 {t[4]:.3f} ms "
                  f"({row['us_per_hyp_iters4']:.1f} us / hypothesis); iters 4 kernels: render {render:.3f} ms, "
                  f"stats + update {fit:.3f} ms", flush=True)
    out["rows"] = rows
    if a.cpu_oracle:
        import translation_oracle as to
        v, f = ro.box()
        mesh = Mesh(v, f)
        R, t_true, masks, _ = scene(mesh, 1, 1, 1)
        render = to.cpu_renderer(v, f, K4, (H, W))
        m = masks[0].cpu().numpy()
        t0 = to.initial_translation(m, K4, diameter(v))
        s = time.perf_counter()
        to.fit(render, R[0], t0, m, K4, 4)
        cpu = 1e3 * (time.perf_counter() - s)
        out["cpu_oracle_box_ms_iters4"] = cpu
        print(f"CPU oracle, box, one hypothesis, iters 4: {cpu:.1f} ms")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
