"""Plain-torch restatement of the joint roll and viewpoint refinement (nope_b200/inplane_refine.py and the
inplane_rotate_pairs / pose_refine_inplane_propose / pose_refine_inplane_select kernels): the rotated pairs, the
proposal of pose and angle slots around each row's centres and the greedy selection over all (angle slot, pose
slot) pairs.  Float32 tensor ops, one rounding per product and per sum, in the kernels' order: the oracle the GPU
tests hold the kernels to bit for bit."""
import itertools
import math

import torch

from oracle import inplane_oracle, refine_oracle

XY, ROLL = 9, 3
XY_OFFSETS = [(0, 0)] + [v for v in itertools.product((-1, 0, 1), repeat=2) if v != (0, 0)]


def xy_stencil(theta):
    """[9, 3, 3] float64: exp([theta * (i, j, 0)]x) by Rodrigues' formula, (0, 0) first, then lexicographic"""
    out = []
    for i, j in XY_OFFSETS:
        phi = theta * math.hypot(i, j)
        if phi == 0.0:
            out.append(torch.eye(3, dtype=torch.float64))
            continue
        x, y = theta * i / phi, theta * j / phi
        K = torch.tensor([[0.0, 0.0, y], [0.0, 0.0, -x], [-y, x, 0.0]], dtype=torch.float64)
        out.append(torch.eye(3, dtype=torch.float64) + math.sin(phi) * K + (1.0 - math.cos(phi)) * (K @ K))
    return torch.stack(out)


def rotate_pairs(images, image_idx, cossin):
    """images [B, 3, H, W], image_idx [P], cossin [P, 2] float32 -> [P, 3, H, W]: pair p is image image_idx[p] rotated
    by cossin[p] with inplane_oracle.rotate's arithmetic, all -1 for an index outside [0, B)"""
    img, idx, cs = images.cpu().float(), image_idx.cpu().long(), cossin.cpu().float()
    B = img.shape[0]
    out = torch.full((idx.shape[0],) + tuple(img.shape[1:]), -1.0)
    for p in range(idx.shape[0]):
        b = int(idx[p])
        if 0 <= b < B:
            out[p] = inplane_oracle.rotate(img[b:b + 1], cs[p:p + 1])[0, 0]
    return out


def compose_roll(cossin, roll_c, roll_s):
    """(c, s) composed with (roll_c, roll_s): (c rc - s rs, s rc + c rs), float32, each op rounded"""
    c, s = cossin[..., 0], cossin[..., 1]
    rc, rs = torch.tensor(roll_c, dtype=torch.float32), torch.tensor(roll_s, dtype=torch.float32)
    return torch.stack([c * rc - s * rs, s * rc + c * rs], dim=-1)


def propose(D, seed, cossin, poses, stencil_, roll, Q):
    """D [R, keep, 9], seed [R, keep], cossin [R, keep, 2], poses [B, N, 6], stencil_ [9, 9], roll (cos, sin) ->
    dict(D, seed, rel [R, keep * 9, 9], poses [R, keep * 9, 6], cossin [R, keep * 3, 2]).  Pose slot c * 9 + j =
    (L_j D_c, seed_c); angle slot c * 3 + l = rho_c, rho_c (+) (cos, sin), rho_c (+) (cos, -sin).  A centre with a
    seed outside [0, N) gives padding pose slots (seed -1, a copy of the row's first valid candidate, I at seed 0 if
    none) and three copies of the first valid centre's rho ((1, 0) if none)."""
    D, seed, poses, stencil_ = D.cpu().float(), seed.cpu().long(), poses.cpu().float(), stencil_.cpu().float()
    cossin = cossin.cpu().float()
    R, keep = seed.shape
    N = poses.shape[1]
    P = keep * XY
    rows = torch.arange(R) // Q
    valid = (seed >= 0) & (seed < N)
    dn = refine_oracle.mat3_mul(stencil_.view(1, 1, XY, 3, 3), D.view(R, keep, 1, 3, 3))
    S = refine_oracle.seed_rotation(poses[rows[:, None], seed.clamp(0, N - 1)])
    rel = refine_oracle.mat3_mul(dn, S[:, :, None])
    out_D, out_rel = dn.reshape(R, P, 9).clone(), rel.reshape(R, P, 9).clone()
    out_seed = torch.where(valid, seed, -1)[:, :, None].expand(R, keep, XY).reshape(R, P).clone()
    c_pos = compose_roll(cossin, roll[0], roll[1])
    c_neg = compose_roll(cossin, roll[0], -roll[1])
    out_cs = torch.stack([cossin, c_pos, c_neg], dim=2)                                  # [R, keep, 3, 2]
    for r in range(R):
        if valid[r].all():
            continue
        if valid[r].any():
            c = int(valid[r].nonzero()[0])
            pd, pr, pc = dn[r, c, 0].reshape(9), rel[r, c, 0].reshape(9), cossin[r, c]
        else:
            eye = torch.eye(3, dtype=torch.float32)
            pd, pr = eye.reshape(9), refine_oracle.mat3_mul(eye, refine_oracle.seed_rotation(poses[rows[r], 0]))
            pr, pc = pr.reshape(9), torch.tensor([1.0, 0.0])
        pad = out_seed[r] < 0
        out_D[r, pad], out_rel[r, pad] = pd, pr
        out_cs[r, ~valid[r]] = pc
    return {"D": out_D, "seed": out_seed.to(torch.int32), "rel": out_rel, "poses": out_rel[..., :6].contiguous(),
            "cossin": out_cs.reshape(R, keep * ROLL, 2).contiguous()}


def rz_mul(cossin, x):
    """Rz(c, s) x over [..., 2] and [..., 9]: rows 1-2 (c x0 - s x1, s x0 + c x1), row 3 copied, float32"""
    c, s = cossin[..., 0:1], cossin[..., 1:2]
    x0, x1, x2 = x[..., 0:3], x[..., 3:6], x[..., 6:9]
    r0, r1 = c * x0 - s * x1, s * x0 + c * x1
    return torch.cat([r0, r1, x2.expand_as(r0)], dim=-1)


def pair_rotations(cand):
    """[R, keep * 3 * keep * 9, 9]: E of every pair m = a * (keep * 9) + p, Rz(rho_a) rel_p"""
    rel, cs = cand["rel"].cpu().float(), cand["cossin"].cpu().float()
    E = rz_mul(cs[:, :, None, :], rel[:, None, :, :])                                    # [R, A3, P, 9]
    return E.reshape(rel.shape[0], -1, 9)


def select(sim, cand, threshold, k):
    """sim [R, keep * 3, keep * 9] at the pairs of propose() -> dict(D [R, k, 9], seed [R, k], cossin [R, k, 2],
    aslot [R, k], score [R, k], rel [R, k, 9]): greedy by descending score, ties -> lowest pair index, pairs with a
    padding pose slot or angle slot never chosen, a pair dropped once trace(E E_b^T) exceeds `threshold` for a chosen
    b; -inf / -1 / zeros past the last pair"""
    R, A3, P = sim.shape
    flat = sim.cpu().float().reshape(R, A3 * P)
    D, seed, rel = cand["D"].cpu().float(), cand["seed"].cpu().long(), cand["rel"].cpu().float()
    cs = cand["cossin"].cpu().float()
    E = pair_rotations(cand)
    out = {"D": torch.zeros((R, k, 9)), "seed": torch.full((R, k), -1, dtype=torch.int32),
           "cossin": torch.zeros((R, k, 2)), "aslot": torch.full((R, k), -1, dtype=torch.int32),
           "score": torch.full((R, k), float("-inf")), "rel": torch.zeros((R, k, 9))}
    thr = torch.tensor(threshold, dtype=torch.float32)
    a_of = torch.arange(A3 * P) // P
    p_of = torch.arange(A3 * P) % P
    for r in range(R):
        alive = (seed[r, p_of] >= 0) & (seed[r, (a_of // ROLL) * XY] >= 0)
        for t in range(k):
            idx = alive.nonzero().flatten()
            if idx.numel() == 0:
                break
            order = torch.sort(-flat[r, idx], stable=True).indices
            m = int(idx[order[0]])
            a, p = m // P, m % P
            out["D"][r, t], out["rel"][r, t], out["cossin"][r, t] = D[r, p], rel[r, p], cs[r, a]
            out["seed"][r, t], out["aslot"][r, t], out["score"][r, t] = int(seed[r, p]), a, flat[r, m]
            alive[m] = False
            alive &= ~(refine_oracle.trace(E[r], E[r, m]) > thr)
    return out
