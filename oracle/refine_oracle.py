"""Plain-torch restatement of the off-grid pose refinement (nope_b200/refine.py and the pose_refine_propose /
pose_refine_select kernels): the lattice stencil, the proposal of candidates around each row's centres and their
greedy selection.  Float32 tensor ops, one rounding per product and per sum, in the kernels' order: the oracle
the GPU tests hold both kernels to bit for bit."""
import itertools
import math

import torch

OFFSETS = [(0, 0, 0)] + [v for v in itertools.product((-1, 0, 1), repeat=3) if v != (0, 0, 0)]


def stencil(theta):
    """[27, 3, 3] float64: exp([theta * v]x) by Rodrigues' formula, v = (0, 0, 0) first, then lexicographic"""
    out = []
    for v in OFFSETS:
        w = torch.tensor(v, dtype=torch.float64) * theta
        phi = float(w.norm())
        if phi == 0.0:
            out.append(torch.eye(3, dtype=torch.float64))
            continue
        x, y, z = (w / phi).tolist()
        K = torch.tensor([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]], dtype=torch.float64)
        out.append(torch.eye(3, dtype=torch.float64) + math.sin(phi) * K + (1.0 - math.cos(phi)) * (K @ K))
    return torch.stack(out)


def mat3_mul(a, b):
    """a @ b over [..., 3, 3] float32: c[i][j] = (a[i][0] b[0][j] + a[i][1] b[1][j]) + a[i][2] b[2][j], every
    product and sum rounded on its own"""
    a, b = torch.broadcast_tensors(a, b)
    c = torch.empty_like(a)
    for i in range(3):
        for j in range(3):
            c[..., i, j] = (a[..., i, 0] * b[..., 0, j] + a[..., i, 1] * b[..., 1, j]) + a[..., i, 2] * b[..., 2, j]
    return c


def seed_rotation(p6):
    """[..., 6] -> [..., 3, 3]: rows 1-2 as given, row 3 = row 1 x row 2"""
    a, b = p6[..., 0:3], p6[..., 3:6]
    c = torch.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], dim=-1)
    return torch.stack([a, b, c], dim=-2)


def propose(D, seed, poses, stencil_, Q):
    """D [R, keep, 9], seed [R, keep], poses [B, N, 6], stencil_ [27, 9] -> dict(D, seed, rel [R, M, 9],
    poses [R, M, 6]), M = keep * 27, slot c * 27 + j = (L_j D_c, seed_c).  A centre with a seed outside [0, N)
    gives padding slots: seed -1, else a copy of the row's first valid candidate (I at seed 0 if none)."""
    D, seed, poses, stencil_ = D.cpu().float(), seed.cpu().long(), poses.cpu().float(), stencil_.cpu().float()
    R, keep = seed.shape
    N = poses.shape[1]
    M = keep * 27
    rows = torch.arange(R) // Q
    valid = (seed >= 0) & (seed < N)
    dn = mat3_mul(stencil_.view(1, 1, 27, 3, 3), D.view(R, keep, 1, 3, 3))                   # [R, keep, 27, 3, 3]
    S = seed_rotation(poses[rows[:, None], seed.clamp(0, N - 1)])                           # [R, keep, 3, 3]
    rel = mat3_mul(dn, S[:, :, None])
    out_D, out_rel = dn.reshape(R, M, 9).clone(), rel.reshape(R, M, 9).clone()
    out_seed = torch.where(valid, seed, -1)[:, :, None].expand(R, keep, 27).reshape(R, M).clone()
    for r in range(R):
        if valid[r].all():
            continue
        if valid[r].any():
            c = int(valid[r].nonzero()[0])
            pd, pr = dn[r, c, 0].reshape(9), rel[r, c, 0].reshape(9)
        else:
            eye = torch.eye(3, dtype=torch.float32)
            pd, pr = eye.reshape(9), mat3_mul(eye, seed_rotation(poses[rows[r], 0])).reshape(9)
        pad = out_seed[r] < 0
        out_D[r, pad], out_rel[r, pad] = pd, pr
    return {"D": out_D, "seed": out_seed.to(torch.int32), "rel": out_rel, "poses": out_rel[..., :6].contiguous()}


def trace(a, b):
    """trace(a b^T) of [..., 9] against [9]: the nine products summed in order, float32"""
    t = a[..., 0] * b[0]
    for e in range(1, 9):
        t = t + a[..., e] * b[e]
    return t


def select(sim, cand, threshold, k):
    """sim [R, M] at the candidates of propose() -> dict(D [R, k, 9], seed [R, k], score [R, k], rel [R, k, 9]):
    greedy by descending score, ties -> lowest slot, padding never chosen, a candidate dropped once its trace
    against a chosen one exceeds `threshold`; -inf / -1 / zeros past the last candidate"""
    sim = sim.cpu().float()
    D, seed, rel = cand["D"].cpu().float(), cand["seed"].cpu().long(), cand["rel"].cpu().float()
    R = sim.shape[0]
    out = {"D": torch.zeros((R, k, 9)), "seed": torch.full((R, k), -1, dtype=torch.int32),
           "score": torch.full((R, k), float("-inf")), "rel": torch.zeros((R, k, 9))}
    thr = torch.tensor(threshold, dtype=torch.float32)
    for r in range(R):
        alive = seed[r] >= 0
        for t in range(k):
            idx = alive.nonzero().flatten()
            if idx.numel() == 0:
                break
            order = torch.sort(-sim[r, idx], stable=True).indices        # slots ascending, so ties -> lowest slot
            m = int(idx[order[0]])
            out["D"][r, t], out["rel"][r, t] = D[r, m], rel[r, m]
            out["seed"][r, t], out["score"][r, t] = int(seed[r, m]), sim[r, m]
            alive[m] = False
            alive &= ~(trace(rel[r], rel[r, m]) > thr)
    return out


def best_score(sim, seed):
    """each row's highest score over its non-padding candidates"""
    return torch.where(seed.cpu() >= 0, sim.cpu(), torch.tensor(float("-inf"))).max(dim=1).values
