"""Time the joint roll and viewpoint refinement against the in-plane search, and measure both on a render-based
stand-in, in ONE process:
  inplane          predict_pose_inplane over level 2 (642 poses) and A angles;
  inplane_refined  predict_pose_inplane_refined from the same search, keep in --keeps, --steps steps.
    python tools/inplane_refine_time.py --queries 1 16 --angles 12 36 --keeps 1 2 --out /tmp/ir.json
Device events around whole calls (encoder included), warm-up of every shape, the cases alternated inside each
repetition; ms is the median over repetitions with the min / max beside it.  Per call and per query row:
`hypotheses` is what the UNet generates (the grid, then keep * 9 per step), `crops` what the encoder encodes (A, then
2 * keep per step).

Accuracy (--standin queries, seeded weights): an engine whose template for a relative pose is the encoder latent of a
render_depth image of an asymmetric mesh (three boxes of distinct sizes) at that pose, the depth shaded into [-1, 1]
and -1 for background, principal point (128, 128) at 256 x 256 (the section 11 convention).  The queries are renders
at seeded off-grid viewpoints with seeded roll.  Reports the median / p90 geodesic error of the in-plane search, of
this refinement, and of the in-plane search chained into refine() on the chosen copy's latent (the existing code
alone).  This describes the seeded encoder on renders; it says nothing about trained weights.  Prints the card name
and power limit with the numbers.  A development aid, not the bench."""
import argparse
import json
import math
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nope_b200 import synth_weights as weights
from nope_b200.inplane import inplane_rotations
from nope_b200.inplane_refine import InplaneRefiner, pose_rotations, refine_inplane
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d, viewpoint_rotations
from nope_b200.refine import PoseRefiner, refine, template_rotations
from nope_b200.vsd import Mesh, render_depth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402

DIST = 400.0                                          # mm, object centre on the optical axis
K_CAM = (300.0, 300.0, 128.0, 128.0)


def geodesic_deg(A, B):
    t = (A.double() * B.double()).sum(dim=(-2, -1))
    return torch.rad2deg(torch.arccos(((t - 1) / 2).clamp(-1, 1)))


def three_boxes():
    """vertices [24, 3] float32 (mm), faces [36, 3] int32: boxes 80 x 24 x 24, 22 x 50 x 18 and 16 x 16 x 44"""
    corners = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    V, F = [], []
    for size, centre in (((80, 24, 24), (0, 0, 0)), ((22, 50, 18), (30, 30, 0)), ((16, 16, 44), (-28, -8, 26))):
        base = len(V)
        V += list(corners * np.array(size) + np.array(centre))
        for a, b, c, d in quads:
            F += [(base + a, base + b, base + c), (base + a, base + c, base + d)]
    return np.array(V, dtype=np.float32), np.array(F, dtype=np.int32)


class RenderEngine:
    """sweep(): the template of relative pose S (rows 1-2 given) is the latent of the mesh rendered at S * ref_R;
    scores are minus the mean squared latent difference (the l2 metric without the occlusion mask)"""

    def __init__(self, encoder, mesh, ref_R):
        self.enc, self.mesh = encoder, mesh
        self.ref_R = torch.as_tensor(ref_R, dtype=torch.float64).cuda()
        self.device = torch.device("cuda:0")

    def images(self, R):
        """object rotations [n, 3, 3] -> shaded renders [n, 3, 256, 256]"""
        T = torch.zeros((R.shape[0], 4, 4), dtype=torch.float64, device=R.device)
        T[:, :3, :3], T[:, 2, 3], T[:, 3, 3] = R, DIST, 1.0
        d = render_depth(self.mesh, T, K_CAM, (256, 256))
        img = torch.where(d > 0, (1.0 - (d - (DIST - 60.0)) / 60.0).clamp(-0.95, 1.0), torch.full_like(d, -1.0))
        return img[:, None].expand(-1, 3, -1, -1).contiguous()

    def templates(self, poses):
        a, b = poses[..., 0:3].double(), poses[..., 3:6].double()
        S = torch.stack([a, b, torch.cross(a, b, dim=-1)], dim=-2)
        flat = (S @ self.ref_R).reshape(-1, 3, 3)
        return torch.cat([self.enc.encode_image(self.images(flat[i:i + 256])) for i in range(0, len(flat), 256)])

    def sweep(self, ref_feat, poses, query_feat=None, want_emb=False, want_sim=True, k=0):
        Rr, M = poses.shape[:2]
        t = self.templates(poses).view(Rr, M, -1)
        q = query_feat if query_feat.dim() == 5 else query_feat[:, None]
        q = q.reshape(Rr, q.shape[1], -1)
        sim = -((q * q).sum(-1)[:, :, None] + (t * t).sum(-1)[:, None, :] - 2 * q @ t.transpose(1, 2)) / q.shape[-1]
        return {"sim": sim if query_feat.dim() == 5 else sim[:, 0], "emb": None, "topv": None, "topi": None}


def accuracy(model, n_q, A, keep, steps, seed=1):
    enc = model.u_net.encoder
    R2 = icosphere_object_rotations(2)
    ref_R = R2[7]
    eng = RenderEngine(enc, Mesh(*three_boxes()), ref_R)
    rel = relative_rotation_6d(R2, ref_R)[None].cuda()
    g = np.random.default_rng(seed)
    gamma = g.uniform(-math.pi, math.pi, n_q)
    Rz = np.stack([[[math.cos(t), -math.sin(t), 0], [math.sin(t), math.cos(t), 0], [0, 0, 1]] for t in gamma])
    qR = torch.from_numpy(Rz @ viewpoint_rotations(g.standard_normal((n_q, 3)))).cuda()
    qimg = eng.images(qR)
    qf = enc.encode_image_inplane(qimg, A)                                           # [n, A, C, 32, 32]
    rf = torch.zeros(1, enc.latent_dim, 32, 32, device=qf.device)
    sim = eng.sweep(rf, rel, qf.view(1, n_q * A, *qf.shape[2:]))["sim"].view(n_q, A, 642)
    flat = torch.sort(-sim.view(n_q, A * 642), dim=1, stable=True).indices[:, :keep]
    n, a = flat % 642, flat // 642
    tp = torch.from_numpy(R2).cuda()
    Rzs = inplane_rotations(A).cuda()
    err = {"inplane": geodesic_deg(Rzs[a[:, 0]] @ tp[n[:, 0]], qR)}
    rows = torch.arange(n_q, device=qf.device)
    lat = qf[rows[:, None], a]
    ir = InplaneRefiner(R2, angles=A, steps=steps)
    out = refine_inplane(eng, enc, rf, qimg[None], rel, (n[None], a[None]), lat[None], ir, k=1)
    err["inplane_refined"] = geodesic_deg(pose_rotations(out["D"], out["seed"], out["cossin"], ir)[0, :, 0], qR)
    # the existing code alone: refine() on the latent of the search's best copy, seeded by that copy's best poses
    a0 = a[:, 0]
    seeds = torch.sort(-sim[rows, a0], dim=1, stable=True).indices[:, :keep]
    pr = PoseRefiner(R2, steps=steps)
    o2 = refine(eng, rf, qf[rows, a0][None], rel, seeds[None], pr, k=1)
    err["inplane+refine"] = geodesic_deg(Rzs[a0] @ template_rotations(o2["D"][0, :, 0], o2["seed"][0, :, 0], pr), qR)
    return {name: (float(e.median()), float(e.quantile(0.9))) for name, e in err.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--angles", type=int, nargs="+", default=[12, 36])
    ap.add_argument("--keeps", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=3, help="calls per timed window")
    ap.add_argument("--standin", type=int, default=32, help="seeded rendered queries for the geodesic error")
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inplane_refine_time.py needs a CUDA device")

    info = card()
    model = build_model(device="cuda:0", precision=args.precision).load_state_dict(
        weights.make_full_state_dict(seed=0)).eval()
    R2 = icosphere_object_rotations(2)
    rel = relative_rotation_6d(R2, R2[7])[None].cuda()
    refiners = {A: InplaneRefiner(R2, angles=A, steps=args.steps) for A in args.angles}
    cases = [("inplane", A, None) for A in args.angles] + \
            [("inplane_refined", A, keep) for A in args.angles for keep in args.keeps]
    g = torch.Generator().manual_seed(0)
    ref = (torch.rand(1, 3, 256, 256, generator=g) * 2 - 1).cuda()
    qry = (torch.rand(max(args.queries), 3, 256, 256, generator=g) * 2 - 1).cuda()

    def call(case, Q):
        name, A, keep = case
        if name == "inplane":
            return lambda: model.predict_pose_inplane(qry[:Q], ref, rel, None, k=5, angles=A)
        return lambda: model.predict_pose_inplane_refined(qry[:Q], ref, rel, refiners[A], k=5, keep=keep)

    fns = {(c, Q): call(c, Q) for c in cases for Q in args.queries}
    for fn in fns.values():
        fn()
        fn()
    samples = {key: [] for key in fns}
    for _ in range(args.reps):
        for Q in args.queries:
            for c in cases:
                samples[(c, Q)].append(timed_ms(fns[(c, Q)], args.iters))

    lines = []
    for Q in args.queries:
        for c in cases:
            name, A, keep = c
            ms = samples[(c, Q)]
            base = samples[(("inplane", A, None), Q)]
            hyps, crops = 642, A
            if keep is not None:
                hyps += refiners[A].hypotheses(keep)
                crops += refiners[A].crops(keep)
            lines.append({"case": name, "A": A, "keep": keep, "steps": args.steps if keep else None, "Q": Q,
                          "precision": args.precision, "hypotheses_per_row": hyps, "crops_per_query": crops,
                          "ms_per_call": round(statistics.median(ms), 3), "ms_min": round(min(ms), 3),
                          "ms_max": round(max(ms), 3),
                          "ms_over_inplane": round(statistics.median(ms) - statistics.median(base), 3), **info})
    for A in args.angles:
        for keep in args.keeps:
            acc = accuracy(model, args.standin, A, keep, args.steps)
            lines.append({"case": "render stand-in accuracy (seeded encoder, not trained weights)", "A": A,
                          "keep": keep, "steps": args.steps, "queries": args.standin,
                          **{f"{k}_median_deg": round(v[0], 3) for k, v in acc.items()},
                          **{f"{k}_p90_deg": round(v[1], 3) for k, v in acc.items()}, **info})
    torch.cuda.synchronize()
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
