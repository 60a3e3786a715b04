"""CPU: the distinct top-k oracle (DESIGN.md section 21) against a plain-Python restatement, the closed form of the
continuous axis against dense sampling, the properties it must have, and every argument refusal of the Python call
and of the C ABI (the library loads without a GPU)."""
import ctypes as C
import math
import os
import zlib

import numpy as np
import pytest
import torch

import distinct_oracle as do
from nope_b200.poses import icosphere_object_rotations

FLIP_Z = np.diag([-1.0, -1.0, 1.0])                                  # 2-fold about z
FLIP_X = np.diag([1.0, -1.0, -1.0])                                  # 2-fold about x
QUARTER_Z = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
GROUPS = {
    "identity": (np.eye(3)[None], np.zeros(3)),
    "flip": (np.stack([np.eye(3), FLIP_Z]), np.zeros(3)),
    "four": (np.stack([np.linalg.matrix_power(QUARTER_Z, i) for i in range(4)]), np.zeros(3)),
    "axis": (np.eye(3)[None], np.array([0.0, 0.0, 1.0])),
    "axis_flip": (np.stack([np.eye(3), FLIP_X]), np.array([0.0, 0.6, 0.8])),
}


def _rand_rot(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3)


def _rodrigues(axis, phi):
    a = np.asarray(axis, np.float64)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + math.sin(phi) * K + (1.0 - math.cos(phi)) * (K @ K)


def _c_scalar(Ri, Rj, D, axis):
    """c(i, j) restated with Python floats, one pair at a time"""
    Ri, Rj = [[float(x) for x in row] for row in Ri], [[float(x) for x in row] for row in Rj]
    P = [[Rj[0][a] * Ri[0][b] + Rj[1][a] * Ri[1][b] + Rj[2][a] * Ri[2][b] for b in range(3)] for a in range(3)]
    ax = [float(x) for x in axis]
    best = None
    for Dd in D:
        Dd = [[float(x) for x in row] for row in Dd]
        M = [[Dd[a][0] * P[0][b] + Dd[a][1] * P[1][b] + Dd[a][2] * P[2][b] for b in range(3)] for a in range(3)]
        t = M[0][0] + M[1][1] + M[2][2]
        if any(ax):
            v = [M[a][0] * ax[0] + M[a][1] * ax[1] + M[a][2] * ax[2] for a in range(3)]
            u = ax[0] * v[0] + ax[1] * v[1] + ax[2] * v[2]
            s = ax[0] * (M[2][1] - M[1][2]) + ax[1] * (M[0][2] - M[2][0]) + ax[2] * (M[1][0] - M[0][1])
            t = u + math.sqrt((t - u) * (t - u) + s * s)
        best = t if best is None else max(best, t)
    return best


def _brute(sim, rot, k, c_thr, D, axis):
    """the greedy loop in plain Python: best remaining (ties -> lowest index), drop what lies within theta"""
    cand = [i for i in range(len(sim)) if sim[i] > -math.inf]
    cand.sort(key=lambda i: (-float(sim[i]), i))
    picked = []
    for i in cand:
        if len(picked) == k:
            break
        if all(_c_scalar(rot[p], rot[i], D, axis) < c_thr for p in picked):
            picked.append(i)
    idx = picked + [-1] * (k - len(picked))
    return np.array([sim[i] if i >= 0 else -np.inf for i in idx], np.float32), np.array(idx, np.int64)


def _grid(golden_dir, name):
    if name == "level1":
        return icosphere_object_rotations(1)
    return np.load(os.path.join(golden_dir, "pose_grids.npz"))[name]


@pytest.mark.parametrize("grid", ["random", "level0_all", "level0_upper", "level1", "level2_all", "level2_upper"])
@pytest.mark.parametrize("group", sorted(GROUPS))
def test_oracle_equals_brute_force(golden_dir, grid, group):
    rng = np.random.default_rng(zlib.crc32(f"{grid} {group}".encode()))
    rot = _rand_rot(rng, 200) if grid == "random" else _grid(golden_dir, grid)
    N = len(rot)
    sim = rng.normal(size=N).astype(np.float32)
    sim[rng.choice(N, N // 4, replace=False)] = sim[rng.choice(N, N // 4)]       # planted exact ties
    sim[rng.choice(N, 3, replace=False)] = -np.inf
    D, axis = GROUPS[group]
    for theta in (0.0, 5.0, 20.0, 90.0):
        k = 12 if N > 300 else 24
        c_thr = do.threshold(theta)
        got = do.distinct_row(sim, rot, k, c_thr, D, axis)
        ref = _brute(sim, rot, k, c_thr, D, axis)
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[0], ref[0]), (theta, got, ref)


def _circle(axis, phis):
    """Rot(a, phi) [P, 3, 3] for every phi (Rodrigues)"""
    a = np.asarray(axis, np.float64)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + np.sin(phis)[:, None, None] * K + (1.0 - np.cos(phis))[:, None, None] * (K @ K)


def test_closed_form_is_the_maximum_over_the_circle():
    """max over phi of tr(M_d Rot(a, phi)) sampled densely, then around the best sample: the closed form is within
    1e-12 of the sampled maximum and never below it"""
    rng = np.random.default_rng(7)
    phis = np.linspace(0.0, 2.0 * math.pi, 20001)
    for D, axis in (GROUPS["axis"], GROUPS["axis_flip"]):
        circle = _circle(axis, phis)
        Ri, Rj = _rand_rot(rng, 40), _rand_rot(rng, 40)
        for i in range(40):
            c = do.closeness(Ri[i], Rj[i:i + 1], D, axis)[0]                              # [n]
            for d in range(len(D)):
                M = D[d] @ Rj[i].T @ Ri[i]
                tr = np.einsum("ij,pji->p", M, circle)
                p0 = phis[int(np.argmax(tr))]
                fine = np.einsum("ij,pji->p", M, _circle(axis, np.linspace(p0 - 4e-4, p0 + 4e-4, 8001))).max()
                dense = max(tr.max(), fine)
                assert c[d] >= dense - 1e-12 and c[d] - dense <= 1e-12, (c[d], dense)


def test_theta_zero_identity_is_plain_topk(golden_dir):
    rng = np.random.default_rng(3)
    rot = _grid(golden_dir, "level2_all")
    sim = np.round(rng.normal(size=len(rot)), 1).astype(np.float32)              # many exact ties
    score, idx = do.distinct_row(sim, rot, 64, do.threshold(0.0), *GROUPS["identity"])
    order = np.argsort(-sim.astype(np.float64), kind="stable")[:64]
    assert np.array_equal(idx, order) and np.array_equal(score, sim[order])


@pytest.mark.parametrize("group", ["flip", "four", "axis", "axis_flip"])
def test_symmetric_copies_are_never_both_selected(group):
    rng = np.random.default_rng(11)
    D, axis = GROUPS[group]
    base = _rand_rot(rng, 30)
    copies = []
    for R in base:                            # Rot_i Rot(a, phi) D_d: the copies bop.symmetry_transformations makes
        for d in range(1, len(D)):
            copies.append(R @ D[d])
        if axis.any():
            copies.append(R @ _rodrigues(axis, rng.uniform(0.1, 6.2)))
            copies.append(R @ _rodrigues(axis, rng.uniform(0.1, 6.2)) @ D[-1])
    rot = np.concatenate([base, np.stack(copies)])
    sim = rng.normal(size=len(rot)).astype(np.float32)
    for theta in (0.01, 0.5, 5.0):        # above the rounding of the copies; theta = 0 in the exact test below
        _, idx = do.distinct_row(sim, rot, 64, do.threshold(theta), D, axis)
        idx = idx[idx >= 0]
        assert len(idx) <= len(base)
        for a in range(len(idx)):
            for b in range(a):
                assert do.closeness(rot[idx[b]], rot[idx[a]][None], D, axis).max() < do.threshold(theta)


def test_symmetric_copy_exact_at_theta_zero():
    """With exactly representable rotations (the 24 rotations of the cube) a copy is caught even at theta = 0"""
    import itertools
    cube = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            M = np.zeros((3, 3))
            M[range(3), perm] = signs
            if np.linalg.det(M) > 0:
                cube.append(M)
    rot = np.stack(cube)
    sim = np.arange(24, dtype=np.float32)[::-1].copy()
    for name, keep in (("identity", 24), ("flip", 12), ("four", 6)):
        _, idx = do.distinct_row(sim, rot, 24, do.threshold(0.0), *GROUPS[name])
        assert (idx >= 0).sum() == keep, name


def test_unscored_entries_and_padding():
    rng = np.random.default_rng(5)
    rot = _rand_rot(rng, 10)
    sim = np.array([1, -np.inf, np.nan, 3, -np.inf, 2, np.nan, np.inf, 0, -1], np.float32)
    score, idx = do.distinct_row(sim, rot, 10, do.threshold(0.0), *GROUPS["identity"])
    assert idx.tolist() == [7, 3, 5, 0, 8, 9, -1, -1, -1, -1]
    assert np.array_equal(score, np.array([np.inf, 3, 2, 1, 0, -1] + [-np.inf] * 4, np.float32))
    # theta = 180 deg: every pair is within, one entry survives
    score, idx = do.distinct_row(sim, rot, 3, do.threshold(180.0), *GROUPS["identity"])
    assert idx.tolist() == [7, -1, -1] and score[1] == -np.inf
    # an all -inf row gives padding only
    score, idx = do.distinct_row(np.full(10, -np.inf, np.float32), rot, 2, 3.0, *GROUPS["identity"])
    assert idx.tolist() == [-1, -1]


def test_symmetry_group_from_models_info(tmp_path):
    from nope_b200 import bop
    from nope_b200.distinct import symmetry_group
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = FLIP_Z, [0.0, 0.0, 5.0]
    (tmp_path / "models_info.json").write_text(
        '{"1": {"diameter": 10.0}, "2": {"diameter": 10.0, "symmetries_discrete": [[%s]]},'
        ' "3": {"diameter": 10.0, "symmetries_continuous": [{"axis": [0, 0, 2], "offset": [0, 0, 0]}],'
        ' "symmetries_discrete": [[%s]]},'
        ' "4": {"diameter": 10.0, "symmetries_continuous": [{"axis": [0, 0, 1]}, {"axis": [1, 0, 0]}]}}'
        % (", ".join(map(repr, T.reshape(-1).tolist())), ", ".join(map(repr, T.reshape(-1).tolist()))))
    info = bop.load_models_info(str(tmp_path / "models_info.json"))
    D, a = symmetry_group(info[1])
    assert np.array_equal(D, np.eye(3)[None]) and not a.any()
    D, a = symmetry_group(info[2])
    assert np.array_equal(D, np.stack([np.eye(3), FLIP_Z])) and not a.any()
    D, a = symmetry_group(info[3])
    assert len(D) == 2 and np.array_equal(a, [0.0, 0.0, 1.0])
    with pytest.raises(ValueError):
        symmetry_group(info[4])
    assert symmetry_group(None)[0].shape == (1, 3, 3)
    with pytest.raises(ValueError):
        symmetry_group({"symmetries_discrete": [np.eye(4)] * 32})


def test_python_argument_errors():
    from nope_b200 import _lib
    from nope_b200.distinct import distinct_topk, threshold
    sim = torch.zeros(2, 6)
    rot = torch.eye(3, dtype=torch.float64).expand(1, 6, 3, 3)
    for bad in (dict(k=0), dict(k=65), dict(k=2.0), dict(k=True), dict(min_angle_deg=-1.0),
                dict(min_angle_deg=181.0), dict(min_angle_deg=float("nan")), dict(min_angle_deg=None),
                dict(sim=sim.double()), dict(sim=sim.numpy()), dict(sim=torch.zeros(2, 0)),
                dict(sim=torch.zeros(1, 1, 1, 6)), dict(rotations=rot[:, :5]), dict(rotations=rot[0]),
                dict(rotations=rot.expand(3, 6, 3, 3)), dict(symmetries=[None] * 3),
                dict(symmetries={"symmetries_continuous": [{"axis": [0, 0, 0]}]})):
        args = dict(sim=sim, rotations=rot, k=2, min_angle_deg=10.0, symmetries=None)
        args.update(bad)
        with pytest.raises(ValueError):
            distinct_topk(**args)
    with pytest.raises(_lib.NopeError):                                          # a valid call on the CPU
        distinct_topk(sim, rot, 2, 10.0, [None, None])
    assert threshold(0) == 3.0 and threshold(180) == -1.0 and threshold(60) == 1.0 + 2.0 * math.cos(math.pi / 3)


def test_c_abi_refusals():
    from nope_b200 import _lib
    lib = _lib.load()
    R, N = 2, 8
    disc = np.concatenate([np.eye(3)[None], FLIP_Z[None]]).astype(np.float64)
    n_disc = np.array([2], np.int32)
    axis = np.zeros((1, 3))
    group = np.zeros(R, np.int32)
    out = C.c_void_p(1)

    def call(**kw):
        a = dict(sim=C.c_void_p(16), R=R, N=N, rot=C.c_void_p(16), G_r=1, Q=1, disc=disc.ctypes.data,
                 n_disc=n_disc.ctypes.data, axis=axis.ctypes.data, G=1, group=group.ctypes.data, k=2, c_thr=2.0,
                 idx=out, score=out)
        a.update(kw)
        return lib.nope_distinct_topk(a["sim"], a["R"], a["N"], a["rot"], a["G_r"], a["Q"], a["disc"], a["n_disc"],
                                      a["axis"], a["G"], a["group"], a["k"], a["c_thr"], a["idx"], a["score"], None)

    held = []

    def nd(*v):
        held.append(np.array(v, np.int32))
        return held[-1].ctypes.data

    def fd(v):
        held.append(np.ascontiguousarray(v, dtype=np.float64))
        return held[-1].ctypes.data

    bad_id = np.concatenate([FLIP_Z[None], np.eye(3)[None]])
    cases = [dict(sim=None), dict(rot=None), dict(disc=None), dict(n_disc=None), dict(axis=None), dict(group=None),
             dict(idx=None), dict(score=None), dict(R=0), dict(N=0), dict(N=(1 << 30) + 1), dict(G_r=0), dict(Q=0),
             dict(G_r=2, Q=2), dict(k=0), dict(k=65), dict(c_thr=3.5), dict(c_thr=-1.5), dict(c_thr=float("nan")),
             dict(G=0), dict(G=65537), dict(n_disc=nd(0)), dict(n_disc=nd(33)), dict(disc=fd(bad_id)),
             dict(disc=fd(np.full((2, 3, 3), np.nan))), dict(axis=fd([[0.0, 0.0, 2.0]])),
             dict(axis=fd([[np.inf, 0.0, 0.0]])), dict(group=nd(0, 1)), dict(group=nd(-1, 0))]
    for case in cases:
        assert call(**case) != 0, case
        assert len(lib.nope_last_error()) > 0
