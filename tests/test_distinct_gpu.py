"""GPU: the distinct top-k kernel (DESIGN.md section 21) against tests/distinct_oracle.py bit for bit, on the rows of
every search (predict_pose at levels 2 and 3 with shared and per-reference template poses, the coarse-to-fine row
with its -inf padding, the in-plane row at A = 36 over 2562 poses) and on a synthetic row above the shared-memory
mask; each row's closeness value pinned to the oracle's last bit; theta = 0 against nope_topk; no host
synchronisation; and select_distinct -> estimate_translation -> eval_bop end to end."""
import math
import os

import numpy as np
import pytest
import torch

import distinct_oracle as do
from _scenes import FLIPS, tless_batch
from _util import no_host_sync

pytestmark = pytest.mark.gpu

B, Q = 2, 4
THETAS = (0.0, 5.0, 20.0, 90.0, 180.0)
FLIP_Z = np.diag([-1.0, -1.0, 1.0])
QUARTER_Z = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])


def _entry(disc=(), axis=None):
    """a bop.load_models_info entry"""
    def T(R):
        m = np.eye(4)
        m[:3, :3] = R
        return m
    return {"diameter": 10.0, "symmetries_discrete": [T(R) for R in disc],
            "symmetries_continuous": [] if axis is None else [{"axis": np.asarray(axis, float), "offset": np.zeros(3)}]}


ENTRIES = {
    "none": _entry(),
    "flip": _entry([FLIP_Z]),
    "four": _entry([np.linalg.matrix_power(QUARTER_Z, i) for i in (1, 2, 3)]),
    "axis_flip": _entry([np.diag([1.0, -1.0, -1.0])], axis=[0.0, 0.0, 3.0]),
}


def _oracle(sim, rot, k, theta, entries):
    """sim [..., N] -> the oracle's (score, idx) in sim's leading shape; entries: None, one entry or one per index of
    sim's first dimension"""
    from nope_b200.distinct import symmetry_group
    s = sim.detach().cpu().numpy()
    lead = s.shape[:-1]
    rows = s.reshape(-1, s.shape[-1])
    first = lead[0] if lead else 1
    if entries is None or isinstance(entries, dict):
        groups, group = [symmetry_group(entries)], [0] * len(rows)
    else:
        groups = [symmetry_group(e) for e in entries]
        group = [r // (len(rows) // first) for r in range(len(rows))]
    r = rot.detach().cpu().numpy().astype(np.float64)
    score, idx = do.distinct_topk(rows, r, k, do.threshold(theta), groups, group, Q=len(rows) // r.shape[0])
    return score.reshape(lead + (k,)), idx.reshape(lead + (k,))


def _check(sim, rot, k, theta, entries):
    from nope_b200.distinct import distinct_topk
    score, idx = distinct_topk(sim, rot, k, theta, entries)
    s_o, i_o = _oracle(sim, rot, k, theta, entries)
    assert np.array_equal(idx.cpu().numpy(), i_o), (k, theta)
    assert np.array_equal(score.cpu().numpy(), s_o), (k, theta)
    return idx


@pytest.fixture(scope="module")
def images():
    from oracle import inputs
    g = torch.Generator().manual_seed(21)
    q = torch.rand(B, Q, 3, 256, 256, generator=g) * 2 - 1
    _, r = inputs.make_images(seed=9, batch=B)
    return q, r


@pytest.fixture(scope="module")
def grids():
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    out = {}
    for level in (2, 3):
        R = torch.from_numpy(icosphere_object_rotations(level))
        out[level] = (R, synthetic_pose_batch(len(R), B)[0].cuda())
    return out


def _per_reference(R):
    """template poses of B references: the grid turned by a different rotation per reference"""
    from scipy.spatial.transform import Rotation
    turn = torch.from_numpy(Rotation.random(B, random_state=4).as_matrix())
    return torch.stack([R @ turn[b] for b in range(B)])


@pytest.mark.parametrize("level", [2, 3])
def test_predict_pose_rows_match_oracle(gpu_model, images, grids, level):
    q, r = images
    R, rel = grids[level]
    _, _, sim = gpu_model.predict_pose(q, r, rel, k=5)                       # [B, Q, N]
    assert sim.shape == (B, Q, len(R))
    shared, per_ref = R[None].cuda(), _per_reference(R).cuda()
    mixed = [ENTRIES["flip"], ENTRIES["axis_flip"]]
    for theta in THETAS:
        for k in (1, 64):
            _check(sim, shared, k, theta, None)
            _check(sim, per_ref, k, theta, mixed)
    for name in ("four", "axis_flip"):
        _check(sim, shared, 64, 20.0, ENTRIES[name])
    _check(sim[:, 0], per_ref, 64, 5.0, mixed)                                # the [B, N] form
    _check(sim[0], shared, 64, 5.0, [ENTRIES["four"]] * Q)                     # the [Q, N] form, per-row groups


def test_theta_zero_identity_equals_nope_topk(gpu_model, images, grids):
    from nope_b200.distinct import distinct_topk
    from nope_b200.model import topk
    q, r = images
    R, rel = grids[2]
    _, _, sim = gpu_model.predict_pose(q, r, rel, k=5)
    sim = torch.round(sim * 4) / 4                                             # exact ties as well
    rows = sim.reshape(-1, sim.shape[-1])
    score, idx = distinct_topk(rows, R[None].cuda(), 64, 0.0)
    v, i = topk(rows, 64)
    assert torch.equal(idx, i) and torch.equal(score, v)


def test_coarse_to_fine_row(gpu_model, images):
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    q, r = images
    Rl = [icosphere_object_rotations(l) for l in range(3)]
    rel = [synthetic_pose_batch(len(x), B)[0].cuda() for x in Rl]
    tp = torch.from_numpy(Rl[2])
    _, _, sim = gpu_model.predict_pose_coarse_to_fine(q, r, rel, PoseHierarchy(Rl), tp, k=5, keep=4)
    unscored = torch.isinf(sim) & (sim < 0)
    assert unscored.float().mean() > 0.5
    for theta in (0.0, 5.0, 20.0):
        idx = _check(sim, tp[None].cuda(), 64, theta, [ENTRIES["none"], ENTRIES["flip"]])
        got = idx.cpu()
        ok = got >= 0
        assert not unscored.cpu().gather(-1, got.clamp_min(0))[ok].any()       # no unscored entry taken
    assert (idx < 0).any()                                                     # padding once the scored run out


def test_inplane_row_and_global_mask(gpu_model, images, grids):
    from nope_b200 import inplane
    from nope_b200.distinct import distinct_topk
    q, r = images
    R, rel = grids[3]
    A, N = 36, len(R)
    _, _, _, sim = gpu_model.predict_pose_inplane(q[:1, :1], r[:1], rel[:1], k=5, angles=A)    # [1, 1, A, N]
    flat = sim.reshape(1, A * N)
    a, n = torch.arange(A).repeat_interleave(N), torch.arange(N).repeat(A)
    rot = inplane.compose(R, n.cuda(), a.cuda(), A)[None]                                     # [1, A N, 3, 3]
    for theta in (5.0, 20.0):
        idx = _check(flat, rot, 64, theta, ENTRIES["flip"])
    got = idx[0].cpu()
    angle, nearest = got // N, got % N
    assert torch.equal(flat[0, idx[0]].cpu(), sim[0, 0][angle, nearest].cpu())
    # above the shared-memory mask (131 072 entries): the masks live in global memory
    g = torch.Generator().manual_seed(5)
    M = 140_000
    big = torch.randn(2, M, generator=g)
    big[:, ::7] = -math.inf
    big[1, 100:200] = big[1, 100]
    from scipy.spatial.transform import Rotation
    rot_big = torch.from_numpy(Rotation.random(2 * M, random_state=6).as_matrix()).reshape(2, M, 3, 3)
    for theta in (0.0, 20.0):
        _check(big.cuda(), rot_big.cuda(), 64, theta, [ENTRIES["none"], ENTRIES["axis_flip"]])
    score, idx = distinct_topk(big.cuda(), rot_big.cuda(), 64, 0.0)
    assert torch.equal(idx, torch.sort(-big, dim=1, stable=True).indices[:, :64].cuda())


def test_closeness_is_bit_exact():
    """Each pair's c(i, j) to the last bit, through the kernel's only decision: with c_thr = the oracle's c the pair
    is suppressed, with the next double above it is not"""
    import ctypes as C
    from nope_b200 import _lib
    from nope_b200.distinct import symmetry_group
    from scipy.spatial.transform import Rotation
    lib = _lib.load()
    rots = Rotation.random(2 * 120, random_state=8).as_matrix().reshape(120, 2, 3, 3)
    sim = torch.tensor([[1.0, 0.0]], device="cuda")
    idx = torch.empty((1, 2), device="cuda", dtype=torch.int64)
    score = torch.empty((1, 2), device="cuda", dtype=torch.float32)
    group = np.zeros(1, np.int32)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    tested = 0
    for name in ("flip", "axis_flip"):
        D, axis = symmetry_group(ENTRIES[name])
        disc, n_disc, ax = np.ascontiguousarray(D), np.array([len(D)], np.int32), np.ascontiguousarray(axis[None])
        for p in range(len(rots)):
            c = do.closeness(rots[p, 0], rots[p, 1][None], D, axis)[0].max()
            if not -1.0 <= c < 3.0:
                continue
            rd = torch.from_numpy(rots[p]).cuda()[None]
            for thr, suppressed in ((c, True), (np.nextafter(c, 4.0), False)):
                _lib.check(lib.nope_distinct_topk(_lib.ptr(sim), 1, 2, _lib.ptr(rd), 1, 1, disc.ctypes.data,
                                                  n_disc.ctypes.data, ax.ctypes.data, 1, group.ctypes.data, 2,
                                                  float(thr), _lib.ptr(idx), _lib.ptr(score), stream))
                assert idx.cpu().tolist() == ([[0, -1]] if suppressed else [[0, 1]]), (name, p, c)
            tested += 1
    assert tested > 200


def test_no_host_synchronisation(grids):
    from nope_b200.distinct import distinct_topk
    R, _ = grids[2]
    rot = R[None].cuda()
    sim = torch.randn(B, Q, len(R), device="cuda")
    with no_host_sync():
        score, idx = distinct_topk(sim, rot, 8, 20.0, [ENTRIES["flip"], ENTRIES["axis_flip"]])
    s_o, i_o = _oracle(sim, rot, 8, 20.0, [ENTRIES["flip"], ENTRIES["axis_flip"]])
    assert np.array_equal(idx.cpu().numpy(), i_o) and np.array_equal(score.cpu().numpy(), s_o)


def test_select_distinct_end_to_end(gpu_model, tmp_path):
    """select_distinct -> estimate_translation -> eval_bop(R_est=, t_est=) on the synthetic T-LESS batch of the BOP
    tests (a box with three flips)"""
    from nope_b200.distinct import distinct_topk
    batch, cad, _ = tless_batch(tmp_path, symmetries=FLIPS)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    info = model.bop_models[1]["info"]
    assert len(info["symmetries_discrete"]) == 3
    _, _, sim = model.predict_pose(batch["query"], batch["reference"], batch["all_relativeR"], k=5)
    tp = batch["template_poses"]
    with pytest.raises(TypeError):
        model.select_distinct(sim, tp, batch["obj_id"], k=5)                 # min_angle_deg has no default
    R, idx, score = model.select_distinct(sim, tp, batch["obj_id"], k=5, min_angle_deg=20.0)
    s2, i2 = distinct_topk(sim, tp, 5, 20.0, [info] * 3)
    assert torch.equal(idx, i2) and torch.equal(score, s2)
    assert R.dtype == torch.float64 and R.shape == (3, 5, 3, 3)
    rows = torch.arange(3)[:, None]
    assert torch.equal(R.cpu(), tp.double()[rows, idx.cpu()])
    masks = torch.stack([torch.from_numpy(np.asarray(
        __import__("cv2").imread(p, -1) > 0)) for p in batch["depth_path"]])
    t, _ = model.estimate_translation(batch, R, masks)
    out = model.eval_bop(batch, "obj01", R_est=R, t_est=t)
    assert sorted(out) == sorted(f"top {k}, {n}" for k in (1, 3, 5) for n in ("ar_vsd", "ar_mssd", "ar_mspd", "ar"))
    # padding rows come back as zero rotations
    R1, idx1, score1 = model.select_distinct(sim, tp, None, k=64, min_angle_deg=90.0)
    pad = idx1 < 0
    assert pad.any() and (R1[pad] == 0).all() and torch.isinf(score1[pad]).all()
    with pytest.raises(ValueError):
        model.select_distinct(sim, tp, [7, 7, 7], k=5, min_angle_deg=20.0)
