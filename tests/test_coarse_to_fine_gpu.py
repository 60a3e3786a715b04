"""GPU: the coarse-to-fine pose search.  The two kernels (pose_cells_expand / pose_cells_rank) against the torch
oracle, bit for bit; whole searches over the synthetic nested icospheres against the exhaustive predict_pose: every
pose the search scores has exactly the exhaustive score, the scored set is the oracle's expansion of the exhaustive
top-`keep`, and the ranking is the exhaustive ranking restricted to that set."""
import pytest
import torch

from _util import no_host_sync
from oracle import hierarchy_oracle as orc

pytestmark = pytest.mark.gpu

B, Q, KEEP, K = 2, 3, 8, 5


@pytest.fixture(scope="module")
def nested():
    """synthetic icosphere levels 0..2 (42 / 162 / 642 poses; level l = first N_l poses of level l + 1), the
    relative rotations of two references at every level, and the hierarchies 162 -> 642 and 42 -> 162 -> 642"""
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    R = [icosphere_object_rotations(l) for l in range(3)]
    rel = {n: synthetic_pose_batch(n, B)[0].cuda() for n in (42, 162, 642)}
    return {"R": R, "rel": rel, "tposes": torch.from_numpy(R[2]),
            "two": PoseHierarchy(R[1:]), "three": PoseHierarchy(R)}


def _rows(t):
    return t.reshape(-1, t.shape[-1]).cpu()


# ------------------------------------------------------------------ kernels
def test_expand_and_rank_kernels_match_oracle(nested):
    from nope_b200.hierarchy import expand, rank
    h = nested["three"]
    cells = h._cells_on(0, "cuda")                     # 42 -> 162
    F = cells.shape[1]
    g = torch.Generator().manual_seed(3)
    keep, M = 6, 6 * F + 5                             # 5 slots beyond keep * F: always padding
    top = torch.randint(-3, 46, (B * Q, keep), generator=g)               # out-of-range entries
    top[0, 3] = top[0, 1]                                                  # repeats
    top[1] = torch.tensor([5, 5, 5, 99, -1, 5])                            # one cell only: fewer than k candidates
    top[2] = -1                                                            # no candidate at all
    poses = torch.randn(B, 162, 6, generator=g)
    cand, p = expand(top.cuda(), cells, poses.cuda(), Q, M)
    cand_o, p_o = orc.expand(top, cells.cpu(), poses, Q, M)
    assert torch.equal(cand.cpu(), cand_o)
    assert torch.equal(p.cpu(), p_o)
    assert (cand_o[1] >= 0).sum() < 10 and (cand_o[2] >= 0).sum() == 0
    sim = torch.randint(-4, 1, (B * Q, M), generator=g).float()            # exact ties everywhere
    for k in (1, 10, 64):
        full, topv, topi = rank(sim.cuda(), cand, 162, k)
        full_o, topv_o, topi_o = orc.rank(sim, cand_o, 162, k)
        assert torch.equal(full.cpu(), full_o), k
        assert torch.equal(topv.cpu(), topv_o), k
        assert torch.equal(topi.cpu(), topi_o), k
        none, topv2, topi2 = rank(sim.cuda(), cand, 162, k, want_sim=False)
        assert none is None and torch.equal(topv2, topv) and torch.equal(topi2, topi)


# ------------------------------------------------------------------ whole searches
@pytest.fixture(scope="module")
def images():
    from oracle import inputs
    g = torch.Generator().manual_seed(21)
    q = torch.rand(B, Q, 3, 256, 256, generator=g) * 2 - 1
    _, r = inputs.make_images(seed=9, batch=B)
    return q, r


@pytest.fixture(scope="module")
def exhaustive(gpu_model, images, nested):
    """predict_pose over each full level: similarity [B, Q, N_l]"""
    q, r = images
    return {n: gpu_model.predict_pose(q, r, nested["rel"][n], k=K)[2] for n in (42, 162, 642)}


@pytest.mark.parametrize("which,sizes", [("two", (162, 642)), ("three", (42, 162, 642))])
def test_search_scores_are_the_exhaustive_scores(gpu_model, images, nested, exhaustive, which, sizes):
    q, r = images
    h = nested[which]
    rel = [nested["rel"][n] for n in sizes]
    R, idx, sim = gpu_model.predict_pose_coarse_to_fine(q, r, rel, h, nested["tposes"], k=K, keep=KEEP)
    assert sim.shape == (B, Q, 642) and idx.shape == (B, Q, K) and R.shape == (B, Q, K, 3, 3)
    ex = exhaustive[642]
    scored = torch.isfinite(sim)
    assert torch.equal(sim[scored], ex[scored])                           # bit-identical where scored
    assert torch.isneginf(sim[~scored]).all()
    cells = [h.cells(s) for s in range(len(sizes) - 1)]
    full, topv, topi, cand = orc.search_from_exhaustive([_rows(exhaustive[n]) for n in sizes], cells, KEEP, K)
    assert torch.equal(_rows(sim), full)
    for row in range(B * Q):                                               # the scored set is the oracle's expansion
        want = set(cand[row][cand[row] >= 0].tolist())
        assert set(torch.nonzero(scored.reshape(B * Q, -1)[row]).flatten().tolist()) == want, row
    assert torch.equal(_rows(idx), topi)
    assert scored.reshape(B * Q, -1).sum(1).max() <= KEEP * cells[-1].shape[1]


def test_search_recovers_a_coarse_pose_template(gpu_model, nested):
    """query feature = the engine's own template at fine pose 5, which every level holds: both searches return
    pose 5 first, with the exhaustive score"""
    from nope_b200.hierarchy import search
    u = gpu_model.u_net
    g = torch.Generator().manual_seed(11)
    rf = (torch.randn(B, 8, 32, 32, generator=g) * 1.5).cuda()
    p = 5
    qf = u.sweep(rf, nested["rel"][642][:, p:p + 1].contiguous(), want_emb=True)["emb"][:, 0]
    ex = u.sweep(rf, nested["rel"][642], query_feat=qf, want_emb=False, k=K)
    assert (ex["topi"][:, 0] == p).all()
    for which, sizes in (("two", (162, 642)), ("three", (42, 162, 642))):
        out = search(u, rf, qf, [nested["rel"][n] for n in sizes], nested[which], keep=KEEP, k=K)
        assert (out["topi"][:, 0] == p).all(), which
        assert torch.equal(out["topv"][:, 0], ex["topv"][:, 0]), which


def test_query_forms_and_R(gpu_model, images, nested):
    q, r = images
    h, tp = nested["two"], nested["tposes"]
    rel = [nested["rel"][162], nested["rel"][642]]
    # [B]: one query per reference
    R, idx, sim = gpu_model.predict_pose_coarse_to_fine(q[:, 0], r, rel, h, tp, k=K, keep=KEEP)
    assert idx.shape == (B, K) and sim.shape == (B, 642)
    assert torch.equal(R.cpu(), tp[idx.cpu()])
    ex = gpu_model.predict_pose(q[:, 0], r, rel[1], k=K)[2]
    assert torch.equal(sim[torch.isfinite(sim)], ex[torch.isfinite(sim)])
    # [Q] against one reference, poses [1, N, 6]
    rel1 = [p[:1] for p in rel]
    R, idx, sim = gpu_model.predict_pose_coarse_to_fine(q[0], r[:1], rel1, h, tp, k=K, keep=KEEP)
    assert idx.shape == (Q, K) and sim.shape == (Q, 642) and R.shape == (Q, K, 3, 3)
    assert torch.equal(R.cpu(), tp[idx.cpu()])
    ex = gpu_model.predict_pose(q[0], r[:1], rel1[1], k=K)[2]
    assert torch.equal(sim[torch.isfinite(sim)], ex[torch.isfinite(sim)])
    full, _, topi, _ = orc.search_from_exhaustive(
        [gpu_model.predict_pose(q[0], r[:1], rel1[0], k=K)[2].cpu(), ex.cpu()], [h.cells(0)], KEEP, K)
    assert torch.equal(sim.cpu(), full) and torch.equal(idx.cpu(), topi)
    # [B, Q]: template_poses [B, N, 3, 3] reads the first reference's grid, as predict_pose does
    R, idx, _ = gpu_model.predict_pose_coarse_to_fine(q, r, rel, h, tp[None].expand(B, -1, -1, -1), k=K, keep=KEEP)
    assert torch.equal(R.cpu(), tp[idx.cpu()])


def test_ldm_search_scores_are_the_exhaustive_scores(nested):
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict
    m = UNetModelPose(device="cuda:0").load_state_dict(make_ldm_state_dict(seed=0))
    g = torch.Generator().manual_seed(5)
    ref = torch.randn(1, 4, 32, 32, generator=g).cuda()
    qry = torch.randn(1, 2, 4, 32, 32, generator=g).cuda()
    from nope_b200.hierarchy import PoseHierarchy
    h = PoseHierarchy(nested["R"][:2])
    rel = [nested["rel"][42][:1], nested["rel"][162][:1]]
    _, idx, sim = m.predict_pose_coarse_to_fine(qry, ref, rel, h, k=K, keep=4)
    ex = [m.predict_pose(qry, ref, p, nested["tposes"][:p.shape[1]], k=K)[2] for p in rel]
    scored = torch.isfinite(sim)
    assert torch.equal(sim[scored], ex[1][scored])
    full, _, topi, _ = orc.search_from_exhaustive([_rows(e) for e in ex], [h.cells(0)], 4, K)
    assert torch.equal(_rows(sim), full) and torch.equal(_rows(idx), topi)


def test_search_does_not_synchronise(gpu_model, nested):
    """The whole search, run after one warm-up call (which reserves the engine workspace and uploads the cell
    tables), under torch's sync debug mode.  That mode sees synchronisation on the Python / torch side only: a
    synchronising call inside the library would not be caught here."""
    from nope_b200.hierarchy import search
    u = gpu_model.u_net
    g = torch.Generator().manual_seed(12)
    rf = torch.randn(B, 8, 32, 32, generator=g).cuda()
    qf = torch.randn(B, Q, 8, 32, 32, generator=g).cuda()
    rel = [nested["rel"][n] for n in (42, 162, 642)]
    ref_out = search(u, rf, qf, rel, nested["three"], keep=KEEP, k=K)
    with no_host_sync():
        out = search(u, rf, qf, rel, nested["three"], keep=KEEP, k=K)
    torch.cuda.synchronize()
    assert torch.equal(out["sim"], ref_out["sim"]) and torch.equal(out["topi"], ref_out["topi"])
    assert out["hypotheses"] == nested["three"].hypotheses(KEEP)
