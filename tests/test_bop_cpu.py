"""CPU: the BOP 2019 host logic -- the models_info parser, symmetry transforms, average recall -- and the numpy oracle of
pose_error_kernel against the textbook formulas."""
import json
import math

import numpy as np
import pytest

from _scenes import FLIPS
from nope_b200 import bop
from oracle import bop_oracle as bo
from oracle import render_oracle as ro


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _pose(rng, z=400.0):
    return np.concatenate([_rot(rng), np.array([[rng.uniform(-30, 30)], [rng.uniform(-30, 30)], [z]])], axis=1)


CYLINDER = {"diameter": 80.0, "symmetries_discrete": [np.diag([1.0, -1.0, -1.0, 1.0])],
            "symmetries_continuous": [{"axis": np.array([0.0, 0.0, 2.0]), "offset": np.array([1.0, -2.0, 0.0])}]}


# ------------------------------------------------------------------ symmetry transforms
@pytest.mark.parametrize("info,count", [({"diameter": 1.0}, 1),
                                        ({"diameter": 1.0, "symmetries_discrete": FLIPS}, 4),
                                        ({"diameter": 1.0, "symmetries_continuous": CYLINDER["symmetries_continuous"]},
                                         315),
                                        (CYLINDER, 630)])
def test_symmetry_transforms_are_rigid_and_counted(info, count):
    T = bop.symmetry_transformations(info)
    D = len(info.get("symmetries_discrete", []))
    n = math.ceil(math.pi / 0.01) if info.get("symmetries_continuous") else 1
    assert n in (1, 315) and T.shape == (count, 3, 4) == ((1 + D) * n, 3, 4)
    R = T[:, :, :3]
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-12
    assert np.abs(np.linalg.det(R) - 1.0).max() < 1e-12
    assert np.array_equal(T[0], np.eye(3, 4))                         # the identity comes first
    assert T.dtype == np.float64


def test_continuous_symmetry_order_angles_and_offset():
    T = bop.symmetry_transformations(CYLINDER)
    n, step = 315, 2 * math.pi / 315
    for i in (1, 7, 314):
        c = T[2 * i]                                                  # continuous i composed with the identity
        ang = math.atan2(c[1, 0], c[0, 0])
        assert abs((ang - i * step + math.pi) % (2 * math.pi) - math.pi) < 1e-12
        off = CYLINDER["symmetries_continuous"][0]["offset"]
        assert np.abs(c[:, :3] @ off + c[:, 3] - off).max() < 1e-12   # the axis through the offset is fixed
        flip = T[2 * i + 1]                                           # ... composed with the discrete flip
        Rd = CYLINDER["symmetries_discrete"][0][:3, :3]
        assert np.abs(flip[:, :3] - c[:, :3] @ Rd).max() < 1e-15
    assert n == len(T) // 2
    finer = bop.symmetry_transformations(CYLINDER, max_sym_disc_step=0.1)
    assert len(finer) == 2 * math.ceil(math.pi / 0.1)


def test_box_flips_map_the_box_onto_itself():
    v, _ = ro.box()
    T = bop.symmetry_transformations({"diameter": 1.0, "symmetries_discrete": FLIPS})
    key = {tuple(p) for p in v.astype(np.float64).tolist()}
    for t in T:
        moved = v.astype(np.float64) @ t[:, :3].T + t[:, 3]
        assert {tuple(p) for p in moved.tolist()} == key
    assert bo.pose_errors_textbook(v, T, np.eye(3, 4)[None] + [[0, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 300]],
                                   (np.eye(3, 4) @ np.diag([1.0, -1, -1, 1]) + [[0, 0, 0, 0], [0, 0, 0, 0],
                                                                                [0, 0, 0, 300]])[None, None],
                                   [[100.0, 100.0, 32.0, 24.0]])[0][0, 0] == 0.0


# ------------------------------------------------------------------ models_info
def test_load_models_info(tmp_path):
    path = tmp_path / "models_info.json"
    path.write_text(json.dumps({
        "1": {"diameter": 63.5, "min_x": -1.0, "symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]},
        "2": {"diameter": 66.2, "symmetries_discrete": [list(np.diag([-1.0, -1, 1, 1]).reshape(-1))]},
        "30": {"diameter": 100.0}}))
    info = bop.load_models_info(str(path))
    assert sorted(info) == [1, 2, 30]
    assert info[1]["diameter"] == 63.5 and info[1]["symmetries_discrete"] == []
    assert np.array_equal(info[1]["symmetries_continuous"][0]["axis"], [0.0, 0.0, 1.0])
    assert np.array_equal(info[2]["symmetries_discrete"][0], np.diag([-1.0, -1, 1, 1]))
    assert info[30]["symmetries_continuous"] == [] and "min_x" not in info[1]
    assert len(bop.symmetry_transformations(info[1])) == 315
    assert len(bop.symmetry_transformations(info[2])) == 2
    assert len(bop.symmetry_transformations(info[30])) == 1
    for bad in ({"x": {"diameter": 1.0}}, {"1": {}}, {"1": {"diameter": -1.0}},
                {"1": {"diameter": 1.0, "symmetries_discrete": [[1, 0, 0]]}},
                {"1": {"diameter": 1.0, "symmetries_continuous": [{"axis": [0, 0, 0], "offset": [0, 0, 0]}]}}):
        path.write_text(json.dumps(bad))
        with pytest.raises(ValueError):
            bop.load_models_info(str(path))


# ------------------------------------------------------------------ average recall
def test_thresholds_are_numpy_arange():
    assert np.array_equal(bop.VSD_TAUS, np.arange(0.05, 0.51, 0.05)) and len(bop.VSD_TAUS) == 10
    assert np.array_equal(bop.MSSD_THETAS, np.arange(0.05, 0.51, 0.05))
    assert np.array_equal(bop.MSPD_THETAS, np.arange(5, 51, 5).astype(np.float64)) and len(bop.MSPD_THETAS) == 10


def test_average_recall_hand_built():
    th = np.arange(0.05, 0.51, 0.05)
    # two targets, one estimate each.  VSD: target 0 scores 0 everywhere (all 100 correct), target 1 scores exactly
    # theta_3 at every tau: correct for the 6 thresholds above it, not at theta_3 itself (strict <)
    vsd = np.stack([np.zeros(10), np.full(10, th[3])])[:, None]
    # MSSD: target 0 exactly at 0.05 x diameter (counts from theta_1), target 1 at 1 mm (always correct)
    diam = np.array([80.0, 50.0])
    mssd = np.array([[th[0] * 80.0], [1.0]])
    # MSPD at W = 1280: thresholds 10, 20, ..., 100 px; target 0 exactly at 10 px, target 1 at 99.99 px
    mspd = np.array([[10.0], [99.99]])
    ar = bop.average_recall(vsd, mssd, mspd, diam, 1280)
    assert ar["ar_vsd"] == (100 + 60) / 200
    assert ar["ar_mssd"] == (9 + 10) / 20
    assert ar["ar_mspd"] == (9 + 1) / 20
    assert ar["ar"] == (ar["ar_vsd"] + ar["ar_mssd"] + ar["ar_mspd"]) / 3
    # k estimates: the per-metric minimum; infinities are never correct
    vsd2 = np.concatenate([np.ones((2, 1, 10)), vsd], axis=1)
    mssd2 = np.concatenate([mssd, np.full((2, 1), np.inf)], axis=1)
    mspd2 = np.concatenate([np.full((2, 1), np.inf), mspd], axis=1)
    assert bop.average_recall(vsd2, mssd2, mspd2, diam, 1280) == ar
    assert bop.average_recall(vsd2[:, :1], mssd2[:, :1], mspd2[:, :1], diam, 1280) == \
        {"ar_vsd": 0.0, "ar_mssd": ar["ar_mssd"], "ar_mspd": 0.0, "ar": ar["ar_mssd"] / 3}
    with pytest.raises(ValueError):
        bop.average_recall(vsd[:, :, :9], mssd, mspd, diam, 1280)
    with pytest.raises(ValueError):
        bop.average_recall(vsd, mssd, mspd, [80.0, 0.0], 1280)


# ------------------------------------------------------------------ oracle vs the textbook formulas
@pytest.mark.parametrize("info", [{"diameter": 1.0}, {"diameter": 1.0, "symmetries_discrete": FLIPS}, CYLINDER])
def test_oracle_matches_textbook(info):
    rng = np.random.default_rng(5)
    pts = rng.normal(0, 30, (200, 3)).astype(np.float32)
    T = bop.symmetry_transformations(info, max_sym_disc_step=0.2)
    gt = np.stack([_pose(rng), _pose(rng, 600.0)])
    est = np.stack([np.stack([_pose(rng), gt[f] + 0.3 * rng.normal(size=(3, 4))]) for f in range(2)])
    K = np.array([[1075.6, 1073.9, 360.0, 270.0], [500.0, 510.0, 320.0, 240.0]])
    ms, mp = bo.pose_errors(pts, T, gt, est, K)
    ts, tp = bo.pose_errors_textbook(pts, T, gt, est, K)
    assert np.abs(ms - ts).max() <= 1e-12 * ts.max()
    assert (np.abs(mp - tp) <= 1e-12 * tp).all()
    assert np.isfinite(ms).all() and np.isfinite(mp).all() and (ms > 0).all()


def test_oracle_behind_camera_is_inf():
    rng = np.random.default_rng(2)
    pts = rng.normal(0, 30, (50, 3)).astype(np.float32)
    gt = _pose(rng)[None]
    est = _pose(rng, -10.0)[None, None]                                # every point behind the camera
    ms, mp = bo.pose_errors(pts, np.eye(3, 4)[None], gt, est, [[100.0, 100.0, 0.0, 0.0]])
    assert np.isfinite(ms).all() and mp[0, 0] == np.inf
