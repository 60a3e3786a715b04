"""Time every greedy selection entry point on its own, at the sizes the searches use:
  nope_topk                        N = 2562 (level 3) and 92 232 (36 in-plane angles x 2562), k = 5 and 64;
  nope_pose_cells_rank             a coarse-to-fine stage into level 3: keep = 64 cells of 8 slots, k = 5 and 64;
  nope_pose_refine_select          M = 64 centres x 27 = 1728 candidates, k = 5 and 64;
  nope_pose_refine_inplane_select  keep = 16: 48 angle slots x 144 pose slots, k = 5 and 64;
  nope_distinct_topk               N = 2562 and 92 232, no symmetry, theta = 20 degrees, k = 5 and 64.
    python tools/rank_time.py --lib nope_b200/lib/libnope_b200.so --lib /path/to/other/libnope_b200.so
Each entry is called on preallocated device buffers (seeded rows, 16 per call), --iters launches back to back between
two CUDA events; the median of --reps such windows is reported per launch.  With several --lib the builds alternate
case by case in one process, so they see the same card state.  Prints the card name and power limit with the
numbers.  A development aid, not the bench."""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402

ROWS = 16


def load(path):
    """a separately bound copy of the library at `path` (several builds can be timed in one process)"""
    _lib._lib, _lib.LIB_PATH = None, os.path.abspath(path)
    lib = _lib.load()
    _lib._lib = None
    return lib


def rotations(n, g):
    """[n, 3, 3] float64 rotations, seeded"""
    q, r = torch.linalg.qr(torch.randn(n, 3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r, dim1=-2, dim2=-1))[:, None, :]
    return q * torch.linalg.det(q)[:, None, None]


def cases(dev):
    """name -> (params, call(lib, stream)) over buffers built once"""
    g = torch.Generator().manual_seed(0)
    P = _lib.ptr
    out = {}
    for N in (2562, 92232):
        sim = torch.randn(ROWS, N, generator=g).to(dev)
        rot = rotations(N, g).to(dev)
        for k in (5, 64):
            topv = torch.empty(ROWS, k, device=dev)
            topi = torch.empty(ROWS, k, device=dev, dtype=torch.int64)
            out[f"topk N={N} k={k}"] = lambda lib, st, sim=sim, k=k, topv=topv, topi=topi, N=N: lib.nope_topk(
                P(sim), ROWS, N, k, P(topv), P(topi), 0, st)
            disc, n_disc = np.eye(3).reshape(1, 9).copy(), np.ones(1, dtype=np.int32)
            axis, group = np.zeros((1, 3)), np.zeros(ROWS, dtype=np.int32)
            c_thr = 1 + 2 * math.cos(math.radians(20.0))
            out[f"distinct N={N} k={k}"] = (
                lambda lib, st, sim=sim, rot=rot, k=k, topv=topv, topi=topi, N=N, disc=disc, n_disc=n_disc,
                axis=axis, group=group, c_thr=c_thr: lib.nope_distinct_topk(
                    P(sim), ROWS, N, P(rot), 1, ROWS, disc.ctypes.data, n_disc.ctypes.data, axis.ctypes.data, 1,
                    group.ctypes.data, k, c_thr, P(topi), P(topv), st))
    # coarse-to-fine stage: 64 disjoint cells of 8 fine poses out of 2562, every 8th slot padding
    n_fine, M = 2562, 64 * 8
    cand = torch.stack([torch.randperm(n_fine, generator=g)[:M] for _ in range(ROWS)]).int()
    cand[:, 7::8] = -1
    cand, csim = cand.to(dev), torch.randn(ROWS, M, generator=g).to(dev)
    out_sim = torch.empty(ROWS, n_fine, device=dev)
    # off-grid refinement: 64 centres x 27; in-plane refinement: 16 centres, 48 angle slots x 144 pose slots
    Mr, keep = 64 * 27, 16
    NP, NA = keep * 9, keep * 3
    thr = 1 + 2 * math.cos(math.radians(2.0))
    ref = {"sim": torch.randn(ROWS, Mr, generator=g), "D": rotations(ROWS * Mr, g).float().reshape(ROWS, Mr, 9),
           "rel": rotations(ROWS * Mr, g).float().reshape(ROWS, Mr, 9),
           "seed": torch.randint(-1, 2562, (ROWS, Mr), generator=g, dtype=torch.int32)}
    inp = {"sim": torch.randn(ROWS, NA * NP, generator=g), "D": rotations(ROWS * NP, g).float().reshape(ROWS, NP, 9),
           "rel": rotations(ROWS * NP, g).float().reshape(ROWS, NP, 9),
           "seed": torch.randint(-1, 2562, (ROWS, NP), generator=g, dtype=torch.int32)}
    a = torch.rand(ROWS, NA, generator=g) * 2 * math.pi
    inp["cossin"] = torch.stack([a.cos(), a.sin()], -1)
    ref, inp = ({n: t.to(dev) for n, t in d.items()} for d in (ref, inp))
    for k in (5, 64):
        topv = torch.empty(ROWS, k, device=dev)
        topi = torch.empty(ROWS, k, device=dev, dtype=torch.int64)
        o = {"D": torch.empty(ROWS, k, 9, device=dev), "rel": torch.empty(ROWS, k, 9, device=dev),
             "seed": torch.empty(ROWS, k, device=dev, dtype=torch.int32), "score": torch.empty(ROWS, k, device=dev),
             "cossin": torch.empty(ROWS, k, 2, device=dev), "aslot": torch.empty(ROWS, k, device=dev, dtype=torch.int32)}
        out[f"cells_rank M={M} k={k}"] = lambda lib, st, k=k, topv=topv, topi=topi: lib.nope_pose_cells_rank(
            P(csim), P(cand), ROWS, M, n_fine, k, P(out_sim), P(topv), P(topi), st)
        out[f"refine_select M={Mr} k={k}"] = lambda lib, st, k=k, o=o: lib.nope_pose_refine_select(
            P(ref["sim"]), P(ref["D"]), P(ref["seed"]), P(ref["rel"]), ROWS, Mr, k, thr, P(o["D"]), P(o["seed"]),
            P(o["score"]), P(o["rel"]), st)
        out[f"inplane_select keep={keep} k={k}"] = lambda lib, st, k=k, o=o: lib.nope_pose_refine_inplane_select(
            P(inp["sim"]), P(inp["D"]), P(inp["seed"]), P(inp["rel"]), P(inp["cossin"]), ROWS, keep, k, thr,
            P(o["D"]), P(o["seed"]), P(o["cossin"]), P(o["aslot"]), P(o["score"]), P(o["rel"]), st)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to time (repeat to alternate builds)")
    ap.add_argument("--iters", type=int, default=200, help="launches per timed window")
    ap.add_argument("--reps", type=int, default=7, help="timed windows per case and library (median)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rank_time.py needs a CUDA device")
    libs = [(p, load(p)) for p in (args.lib or [_lib.LIB_PATH])]
    dev = torch.device("cuda:0")
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    info = card()
    lines = []
    for name, call in cases(dev).items():
        ms = {p: [] for p, _ in libs}
        for _, lib in libs:                                           # warm-up, and any refusal surfaces here
            rc = call(lib, st)
            if rc != 0:
                raise SystemExit(f"{name}: {lib.nope_last_error().decode()}")
        for _ in range(args.reps):
            for p, lib in libs:
                ms[p].append(timed_ms(lambda: call(lib, st), args.iters))
        for p, _ in libs:
            line = {"case": name, "lib": p, "ms": round(statistics.median(ms[p]), 5),
                    "min_ms": round(min(ms[p]), 5), "max_ms": round(max(ms[p]), 5), "rows": ROWS, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
