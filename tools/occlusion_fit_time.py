"""Measure the pose fits under occlusion (DESIGN.md section 24) at 720x540 with the Primesense intrinsics.

--accuracy: 32 seeded scenes per mesh (box, icosphere) and occlusion level (a nearer sphere hiding 20, 40 or 60 % of
the target's silhouette; tests/_scenes.occluded_scene), with the visible mask M and the occluders O.
For the translation fit from initial_translation(M) at the true rotation: median / max |dz| in box pixels
(|dz| sqrt(w h) / z, with the box of the whole silhouette) and the origin's reprojection error in px after 0 ... 6
updates, with and without O.  For the contour refinement from starts 2.5 - 5 deg and 5 - 10 mm off: median / max
translation (mm) and rotation (deg) error after the default schedule, with and without O.

Timing: both fits at F in {1, 16} frames, P = 5 hypotheses, the default iterations, for the box and a 20 480-triangle
icosphere, with and without O: CUDA events around the Python call, median of --reps.  The card's name and power limit
are read in the same run.

    python tools/occlusion_fit_time.py [--reps 20] [--accuracy] [--scenes 32]
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

from _scenes import K4, accuracy, occluded_scene, perturb                      # noqa: E402
from nope_b200.contour_refine import refine_pose_contour                       # noqa: E402
from nope_b200.translation import DEFAULT_ITERS, estimate_translation          # noqa: E402
from nope_b200.vsd import Mesh                                                 # noqa: E402
from oracle import render_oracle as ro                                         # noqa: E402
from translation_time import card, timed                                       # noqa: E402

LEVELS = (0.2, 0.4, 0.6)


def _diameter(v):
    return float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))


def accuracy_table(n):
    rows = []
    for name, (v, f) in {"box": ro.box(), "icosphere": ro.sphere(40.0, 2)}.items():
        mesh, d = Mesh(v, f), _diameter(v)
        for cover in LEVELS:
            for it in range(7):
                e = accuracy(mesh, d, name, cover, n, iters=it)
                for key in ("O", "no O"):
                    r = {"mesh": name, "cover": cover, "occluders": key, "iters": it}
                    cols = ("dz_px", "reproj_px") if it != DEFAULT_ITERS else ("dz_px", "reproj_px", "t_mm", "r_deg")
                    for c in cols:
                        r[c + "_med"], r[c + "_max"] = float(np.median(e[key][c])), float(np.max(e[key][c]))
                    rows.append(r)
                    print(" ".join(f"{k}={x:.3f}" if isinstance(x, float) else f"{k}={x}" for k, x in r.items()),
                          flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scenes", type=int, default=32)
    ap.add_argument("--accuracy", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("occlusion_fit_time.py needs a CUDA GPU")
    name, pl = card()
    print(f"# {name}, power limit {pl}; 720x540, P = 5; CUDA events, median of {a.reps}")
    out = {"card": name, "power_limit": pl}
    if a.accuracy:
        out["accuracy"] = accuracy_table(a.scenes)
    rows, P = [], 5
    for mname, (v, f) in {"box (12)": ro.box(), "icosphere (20480)": ro.sphere(40.0, 5)}.items():
        mesh = Mesh(v, f)
        for F in (1, 16):
            R_true, t_true, M, O, *_ = occluded_scene(mesh, 1, F, 0.4)
            rng = np.random.default_rng(2)
            st = [[perturb(rng, R_true[i], t_true[i]) for _ in range(P)] for i in range(F)]
            Rd = torch.from_numpy(np.array([[s[0] for s in r] for r in st])).cuda()
            td = torch.from_numpy(np.array([[s[1] for s in r] for r in st])).cuda()
            for occ_name, occ in (("no O", None), ("O", O)):
                ms_t = timed(lambda: estimate_translation(mesh, Rd, K4, M, t_init=td, occluders=occ), a.reps)
                ms_c = timed(lambda: refine_pose_contour(mesh, Rd, td, K4, M, occluders=occ), a.reps)
                rows.append({"mesh": mname, "F": F, "P": P, "occluders": occ_name, "translation_ms": ms_t,
                             "contour_ms": ms_c})
                print(f"{mname:18s} F {F:2d} {occ_name:4s}: translation {ms_t:.3f} ms, contour {ms_c:.3f} ms",
                      flush=True)
    out["rows"] = rows
    print(json.dumps(out))


if __name__ == "__main__":
    main()
