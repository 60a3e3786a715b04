"""CPU: the coarse-to-fine pose search without a device -- cell tables on the reference's shipped grids and on the
synthetic nested icospheres, the torch oracle's expand / rank conventions and the Python argument
errors."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import hierarchy_oracle as orc


@pytest.fixture(scope="module")
def grids(golden_dir):
    g = np.load(os.path.join(golden_dir, "pose_grids.npz"))
    n = np.load(os.path.join(golden_dir, "pose_nesting.npz"))
    return {k: g[k] for k in g.files}, {k: n[k] for k in n.files}


def _check_partition(table, n_fine):
    """cells are disjoint, cover the fine grid, ascending, and -1 padded after the last entry; F is the largest"""
    assert table.dtype == np.int32
    counts = (table >= 0).sum(axis=1)
    assert table.shape[1] == counts.max()
    for row, n in zip(table, counts):
        assert (row[:n] >= 0).all() and (row[n:] == -1).all()
        assert (np.diff(row[:n]) > 0).all()
    flat = table[table >= 0]
    assert np.array_equal(np.sort(flat), np.arange(n_fine))


@pytest.mark.parametrize("dist", ["all", "upper"])
def test_reference_nesting_lies_in_own_cell(grids, dist):
    """level 0 against the level-2 'all' grid: each coarse pose's nearest fine pose is the reference's
    idx_{dist}_level0_in_level2[i] and belongs to coarse pose i's own cell"""
    from nope_b200.hierarchy import cell_table, rotation_trace
    g, nest = grids
    coarse, fine = g[f"level0_{dist}"], g["level2_all"]
    idx = nest[f"idx_{dist}_level0_in_level2"]
    assert idx.shape == (coarse.shape[0],)
    assert np.array_equal(np.argmax(rotation_trace(fine, coarse), axis=0), idx)
    table = cell_table(coarse, fine)
    _check_partition(table, fine.shape[0])
    for i, f in enumerate(idx):
        assert f in table[i], (i, f)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_synthetic_nested_grids(level):
    """level l is the first N_l vertices of level l + 1: coarse pose i's cell holds fine pose i"""
    from nope_b200.hierarchy import cell_table
    from nope_b200.poses import icosphere_object_rotations
    c, f = icosphere_object_rotations(level), icosphere_object_rotations(level + 1)
    assert np.array_equal(f[:len(c)], c)
    table = cell_table(c, f)
    _check_partition(table, f.shape[0])
    for i in range(len(c)):
        assert i in table[i]
    assert table.shape[1] <= 7


def test_product_table_equals_oracle(grids):
    """the product's numpy cell table and the oracle's torch restatement agree, exact ties included"""
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.poses import icosphere_object_rotations
    g, _ = grids
    h = PoseHierarchy([g["level0_all"], g["level2_all"]])
    assert torch.equal(h.cells(0), orc.cell_table(g["level0_all"], g["level2_all"]))
    levels = [icosphere_object_rotations(l) for l in range(3)]
    h = PoseHierarchy(levels)
    assert h.sizes == (42, 162, 642)
    for s in range(2):
        assert torch.equal(h.cells(s), orc.cell_table(levels[s], levels[s + 1]))
    assert h.hypotheses(8) == 42 + 8 * h.cell_width(0) + 8 * h.cell_width(1)


def test_oracle_expand_order_and_padding():
    cells = torch.tensor([[0, 3, -1], [1, -1, -1], [2, 4, 5]], dtype=torch.int32)
    poses = torch.arange(2 * 6 * 6, dtype=torch.float32).reshape(2, 6, 6)
    top = torch.tensor([[2, 0, 2, 7], [-1, 1, 9, 1], [-3, 5, 3, 4]])       # repeats and out-of-range entries
    cand, p = orc.expand(top, cells, poses, Q=3, M=12)                    # rows 0..2: reference 0
    assert cand[0].tolist() == [2, 4, 5, 0, 3] + [-1] * 7                  # top_idx order, ascending in a cell
    assert cand[1].tolist() == [1] + [-1] * 11
    assert cand[2].tolist() == [-1] * 12
    assert torch.equal(p[0, :5], poses[0, [2, 4, 5, 0, 3]])
    assert torch.equal(p[0, 5:], poses[0, 2].expand(7, 6))                 # padding: the row's first candidate
    assert torch.equal(p[2], poses[0, 0].expand(12, 6))                    # no candidate: fine pose 0
    cand, p = orc.expand(top[:2], cells, poses, Q=1, M=12)                  # Q = 1: row 1 is reference 1
    assert torch.equal(p[1, 0], poses[1, 1])


def test_oracle_rank_ties_and_padding():
    sim = torch.tensor([[1.0, 3.0, 3.0, 2.0, 9.0], [5.0, 5.0, 0.0, 0.0, 0.0]])
    cand = torch.tensor([[7, 4, 2, 9, -1], [3, 1, -1, -1, -1]], dtype=torch.int32)
    full, topv, topi = orc.rank(sim, cand, 10, 4)
    assert topi.tolist() == [[2, 4, 9, 7], [1, 3, -1, -1]]                  # equal scores: lowest fine index first
    assert topv[0].tolist() == [3.0, 3.0, 2.0, 1.0]
    assert topv[1, :2].tolist() == [5.0, 5.0] and torch.isneginf(topv[1, 2:]).all()
    assert full[0, 7] == 1.0 and full[0, 2] == 3.0 and torch.isneginf(full[0, [0, 1, 3, 5, 6, 8]]).all()
    assert torch.isneginf(full[1]).sum() == 8


@pytest.mark.parametrize("args,needle", [
    (dict(R=2, keep=0, F=3, B=2, Q=1, M=6), "keep"),
    (dict(R=2, keep=65, F=3, B=2, Q=1, M=300), "keep"),
    (dict(R=2, keep=2, F=3, B=2, Q=1, M=5), "M"),
    (dict(R=3, keep=2, F=3, B=2, Q=1, M=6), "R"),
])
def test_expand_rejects_bad_sizes(args, needle):
    import ctypes as C
    from nope_b200 import _lib
    lib = _lib.load()
    p = C.c_void_p(256)
    rc = lib.nope_pose_cells_expand(p, args["R"], args["keep"], p, 10, args["F"], p, args["B"], args["Q"], 40,
                                    args["M"], p, p, None)
    assert rc != 0 and needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("k", [0, 65])
def test_rank_rejects_bad_k(k):
    import ctypes as C
    from nope_b200 import _lib
    lib = _lib.load()
    p = C.c_void_p(256)
    assert lib.nope_pose_cells_rank(p, p, 2, 8, 40, k, None, p, p, None) != 0
    assert "k" in lib.nope_last_error().decode()


def _levels(B=1):
    from nope_b200.poses import icosphere_object_rotations
    R = [icosphere_object_rotations(l) for l in (0, 1)]
    return R, [torch.zeros(B, len(r), 6) for r in R]


def test_python_argument_errors_without_a_device():
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.ldm import UNetModelPose
    from nope_b200.model import PoseConditional
    R, rel = _levels()
    with pytest.raises(ValueError):
        PoseHierarchy(R[:1])
    h = PoseHierarchy(R)
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    ldm = UNetModelPose(device="cpu")
    img, lat = torch.zeros(1, 3, 256, 256), torch.zeros(1, 4, 32, 32)
    bad = [dict(all_relativeR_levels=rel[:1]),                              # fewer than two levels
           dict(all_relativeR_levels=[rel[0], torch.zeros(1, 161, 6)]),      # N_l mismatch
           dict(all_relativeR_levels=rel, keep=43),                          # keep > N_0
           dict(all_relativeR_levels=rel, keep=0),
           dict(all_relativeR_levels=rel, k=0),
           dict(all_relativeR_levels=rel, k=65)]
    for kw in bad:
        kw = {"hierarchy": h, **kw}
        with pytest.raises(ValueError):
            model.predict_pose_coarse_to_fine(img, img, **kw)
        with pytest.raises(ValueError):
            ldm.predict_pose_coarse_to_fine(lat, lat, **kw)


def test_sharded_model_is_refused():
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.model import PoseConditional
    R, rel = _levels()
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    model.dist = object()
    img = torch.zeros(1, 3, 256, 256)
    with pytest.raises(NotImplementedError, match="shard"):
        model.predict_pose_coarse_to_fine(img, img, rel, PoseHierarchy(R))
