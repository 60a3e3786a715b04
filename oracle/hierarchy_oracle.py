"""Plain-torch restatement of the coarse-to-fine pose search (nope_b200/hierarchy.py and the
pose_cells_expand / pose_cells_rank kernels): the cell table, the expansion of a row's kept coarse poses into
the union of their cells, and the ranking of the scored candidates.  Loops and sorts, no kernels: the oracle the
GPU tests hold both kernels and the whole search to."""
import torch


def rotation_trace(fine_R, coarse_R):
    """trace(R_f R_c^T) [N_fine, N_coarse], float64, the nine products summed left to right"""
    f = torch.as_tensor(fine_R, dtype=torch.float64).reshape(-1, 1, 9)
    c = torch.as_tensor(coarse_R, dtype=torch.float64).reshape(1, -1, 9)
    p = f * c
    t = p[..., 0].clone()
    for j in range(1, 9):
        t = t + p[..., j]
    return t


def cell_table(coarse_R, fine_R):
    """int32 [N_coarse, F]: the fine poses nearest (largest trace, ties -> lowest coarse index) to each coarse pose,
    ascending, -1 padded; F = the largest cell"""
    nearest = rotation_trace(fine_R, coarse_R).argmax(dim=1)          # first maximum = lowest coarse index
    n_coarse = torch.as_tensor(coarse_R).shape[0]
    cells = [[f for f in range(nearest.shape[0]) if int(nearest[f]) == i] for i in range(n_coarse)]
    F = max(len(c) for c in cells)
    out = torch.full((n_coarse, F), -1, dtype=torch.int32)
    for i, c in enumerate(cells):
        out[i, :len(c)] = torch.tensor(c, dtype=torch.int32)
    return out


def expand(top_idx, cells, poses, Q, M):
    """top_idx [R, keep] int64, cells [N_coarse, F], poses [B, n_fine, 6] -> (cand [R, M] int32, poses [R, M, 6]).
    Kept entries in order, skipping indices outside [0, N_coarse) and repeats; each cell ascending; -1 after the
    last candidate; a padding slot carries the row's first candidate pose (fine pose 0 if there is none)."""
    top_idx, cells, poses = top_idx.cpu(), cells.cpu(), poses.cpu()
    R = top_idx.shape[0]
    n_coarse = cells.shape[0]
    cand = torch.full((R, M), -1, dtype=torch.int32)
    out = torch.empty((R, M, 6), dtype=poses.dtype)
    for r in range(R):
        seen, fine = set(), []
        for c in top_idx[r].tolist():
            if c < 0 or c >= n_coarse or c in seen:
                continue
            seen.add(c)
            fine += [f for f in cells[c].tolist() if f >= 0]
        cand[r, :len(fine)] = torch.tensor(fine, dtype=torch.int32)
        pad = fine[0] if fine else 0
        out[r] = poses[r // Q, [f if f >= 0 else pad for f in cand[r].tolist()]]
    return cand, out


def rank(sim, cand, n_fine, k):
    """sim [R, M] scored at cand [R, M] -> (sim over the fine grid [R, n_fine], -inf where not scored;
    topv [R, k]; topi [R, k] int64): descending score, ties -> lowest fine index, -inf / -1 past the candidates"""
    sim, cand = sim.cpu(), cand.cpu().long()
    R = sim.shape[0]
    full = torch.full((R, n_fine), float("-inf"), dtype=sim.dtype)
    topv = torch.full((R, k), float("-inf"), dtype=sim.dtype)
    topi = torch.full((R, k), -1, dtype=torch.int64)
    for r in range(R):
        ok = cand[r] >= 0
        idx, val = cand[r][ok], sim[r][ok]
        full[r, idx] = val
        by_index = torch.argsort(idx)                                    # fine index ascending ...
        idx, val = idx[by_index], val[by_index]
        order = torch.sort(-val, stable=True).indices[:k]                # ... then descending score, stable
        topv[r, :len(order)] = val[order]
        topi[r, :len(order)] = idx[order]
    return full, topv, topi


def topk_lowest_index(sim, k):
    """descending score, ties -> lowest index"""
    order = torch.sort(-sim, dim=1, stable=True).indices[:, :k]
    return sim.gather(1, order), order


def search_from_exhaustive(sims, cells, keep, k, Q=1):
    """The search restated over exhaustive similarities: sims[l] [R, N_l] is every pose of level l scored for each
    row, cells[l] the table of the step l -> l + 1.  Each stage keeps the top `keep` of the poses the previous stage
    expanded to -- exactly what the search does when a pose's score does not depend on the other poses of its
    launch.  -> (sim [R, N_L] with -inf where not scored, topv [R, k], topi [R, k], cand [R, M] of the last stage)"""
    sims = [s.cpu() for s in sims]
    _, top = topk_lowest_index(sims[0], keep)
    R = sims[0].shape[0]
    for l in range(1, len(sims)):
        F = cells[l - 1].shape[1]
        dummy = torch.zeros((R, sims[l].shape[1], 6))
        cand, _ = expand(top, cells[l - 1], dummy, 1, keep * F)
        scored = torch.where(cand >= 0, sims[l].gather(1, cand.clamp_min(0).long()),
                             torch.zeros((), dtype=sims[l].dtype))
        full, topv, top = rank(scored, cand, sims[l].shape[1], k if l == len(sims) - 1 else keep)
    return full, topv, top, cand
