"""GPU: the BOP 2019 errors.  pose_error_kernel against the numpy oracle bit for bit (symmetry counts 1 ... 630, point
counts 1 ... 40 000, points behind the camera), launch-shape and batch independence, exact cases (est = gt, a symmetric
estimate, a pure translation error, a rotation about a continuous axis), multi-tau VSD against single-tau VSD and the
reference's values, and eval_bop end to end on a synthetic T-LESS batch."""
import math
import os

import numpy as np
import pytest
import torch

from _scenes import FLIPS, K4, tless_batch
from _util import no_host_sync
from oracle import bop_oracle as bo
from oracle import render_oracle as ro

pytestmark = pytest.mark.gpu

CYL = {"diameter": 80.0, "symmetries_discrete": [np.diag([1.0, -1.0, -1.0, 1.0])],
       "symmetries_continuous": [{"axis": np.array([0.0, 0.0, 1.0]), "offset": np.array([0.0, 0.0, 0.0])}]}


def _rot(rng, scale=math.pi):
    w = rng.normal(size=3)
    w = w / np.linalg.norm(w) * rng.uniform(0, scale)
    from nope_b200.bop import _rodrigues
    return _rodrigues(w, np.linalg.norm(w)) if np.linalg.norm(w) > 0 else np.eye(3)


def _pose(rng, z=500.0):
    return np.concatenate([_rot(rng), [[rng.uniform(-40, 40)], [rng.uniform(-40, 40)], [z]]], axis=1)


def _syms(S):
    from nope_b200 import bop
    if S == 1:
        return np.eye(3, 4)[None]
    if S == 2:
        return bop.symmetry_transformations({"symmetries_discrete": FLIPS[:1]})
    if S == 315:
        return bop.symmetry_transformations({"symmetries_continuous": CYL["symmetries_continuous"]})
    return bop.symmetry_transformations(CYL)


def _run(pts, syms, gt, est, K):
    from nope_b200.bop import pose_errors
    ms, mp = pose_errors(torch.from_numpy(pts).cuda(), torch.from_numpy(est[..., :3]), torch.from_numpy(est[..., 3]),
                         torch.from_numpy(gt[..., :3]), torch.from_numpy(gt[..., 3]), K, syms)
    return ms.cpu().numpy(), mp.cpu().numpy()


def _case(seed, V, F, P, behind=False):
    rng = np.random.default_rng(seed)
    pts = rng.normal(0, 30, (V, 3)).astype(np.float32)
    gt = np.stack([_pose(rng, rng.uniform(300, 900)) for _ in range(F)])
    est = np.stack([np.stack([_pose(rng, rng.uniform(300, 900)) for _ in range(P)]) for _ in range(F)])
    if behind:
        est[0, 0, 2, 3] = 10.0                                      # some points behind the camera
        gt[-1, 2, 3] = -5.0                                         # the ground truth too, for one row
    K = np.stack([K4 * [1, 1, 1 + 0.1 * f, 1] for f in range(F)])
    return pts, gt, est, K


# ------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("S", [1, 2, 315, 630])
@pytest.mark.parametrize("V,F,P", [(1, 1, 1), (31, 2, 3), (1000, 3, 2), (40000, 1, 1)])
def test_pose_errors_match_oracle(S, V, F, P):
    pts, gt, est, K = _case(S * 7 + V, V, F, P)
    syms = _syms(S)
    ms, mp = _run(pts, syms, gt, est, K)
    rs, rp = bo.pose_errors(pts, syms, gt, est, K)
    assert np.array_equal(ms, rs) and np.array_equal(mp, rp), (ms, rs, mp, rp)
    assert np.isfinite(ms).all()


def test_points_behind_the_camera():
    pts, gt, est, K = _case(11, 500, 3, 2, behind=True)
    syms = _syms(630)
    ms, mp = _run(pts, syms, gt, est, K)
    rs, rp = bo.pose_errors(pts, syms, gt, est, K)
    assert np.array_equal(ms, rs) and np.array_equal(mp, rp)
    assert mp[0, 0] == np.inf and (mp[-1] == np.inf).all() and np.isfinite(mp[1]).all() and np.isfinite(ms).all()


def test_launch_split_and_batch_composition():
    pts, gt, est, K = _case(3, 3000, 4, 5)
    syms = _syms(630)
    ms, mp = _run(pts, syms, gt, est, K)
    # symmetry subsets whose sizes are not multiples of the per-CTA chunk: the min over the parts is the whole
    parts = [_run(pts, syms[a:b], gt, est, K) for a, b in ((0, 1), (1, 314), (314, 630))]
    assert np.array_equal(np.minimum.reduce([p[0] for p in parts]), ms)
    assert np.array_equal(np.minimum.reduce([p[1] for p in parts]), mp)
    for f in range(4):                                              # one row alone, one estimate alone
        a, b = _run(pts, syms, gt[f:f + 1], est[f:f + 1], K[f:f + 1])
        assert np.array_equal(a, ms[f:f + 1]) and np.array_equal(b, mp[f:f + 1])
        a, b = _run(pts, syms, gt[f:f + 1], est[f:f + 1, 2:3], K[f:f + 1])
        assert np.array_equal(a, ms[f:f + 1, 2:3]) and np.array_equal(b, mp[f:f + 1, 2:3])
    perm = np.random.default_rng(0).permutation(len(pts))           # point order
    a, b = _run(pts[perm], syms, gt, est, K)
    assert np.array_equal(a, ms) and np.array_equal(b, mp)


# ------------------------------------------------------------------ exact cases
def test_est_equal_gt_and_symmetric_estimates():
    pts, gt, _, K = _case(4, 2000, 2, 1)
    syms = _syms(630)
    ms, mp = _run(pts, syms, gt, gt[:, None], K)
    assert (ms == 0).all() and (mp == 0).all()
    diameter = float(np.max(np.linalg.norm(pts[:, None].astype(np.float64) - pts[None], axis=2)))
    for j in (1, 2, 101, 629):
        Rs, ts = syms[j, :, :3], syms[j, :, 3]
        est = np.concatenate([gt[:, :, :3] @ Rs, (gt[:, :, :3] @ ts + gt[:, :, 3])[..., None]], axis=2)[:, None]
        ms, mp = _run(pts, syms, gt, est, K)
        assert (ms <= 1e-9 * diameter).all(), (j, ms)


def test_pure_translation_error():
    pts, gt, _, K = _case(5, 3000, 2, 1)
    dt = np.array([3.0, -4.0, 12.0])
    est = gt.copy()
    est[:, :, 3] += dt
    ms, _ = _run(pts, np.eye(3, 4)[None], gt, est[:, None], K)
    assert np.abs(ms - 13.0).max() < 1e-9


def test_rotation_about_a_continuous_axis():
    """a rotation about the symmetry axis: within the discretisation bound of a cylinder; the same object declared
    asymmetric is far off"""
    rng = np.random.default_rng(6)
    pts = rng.normal(0, 25, (2000, 3)).astype(np.float32)
    radius = float(np.linalg.norm(pts[:, :2], axis=1).max())
    gt = _pose(rng)[None]
    for ang in (0.004, 0.3, 1.0, 2.9):
        c, s = math.cos(ang), math.sin(ang)
        Rz = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        est = np.concatenate([gt[:, :, :3] @ Rz, gt[:, :, 3:]], axis=2)[:, None]
        sym, _ = _run(pts, _syms(315), gt, est, K4[None])
        asym, _ = _run(pts, _syms(1), gt, est, K4[None])
        bound = 2 * radius * math.sin(math.pi / 315 / 2)            # half a step of 2 pi / 315
        assert sym[0, 0] <= bound + 1e-9
        exact = 2 * radius * math.sin(ang / 2)
        assert abs(asym[0, 0] - exact) < 1e-6 * exact and (ang < 0.01 or asym[0, 0] > 10 * bound)


def test_pose_errors_bad_arguments_and_no_sync():
    from nope_b200 import _lib
    from nope_b200.bop import pose_errors
    pts, gt, est, K = _case(8, 100, 2, 2)
    args = (torch.from_numpy(pts).cuda(), torch.from_numpy(est[..., :3]).cuda(), torch.from_numpy(est[..., 3]).cuda(),
            torch.from_numpy(gt[..., :3]).cuda(), torch.from_numpy(gt[..., 3]).cuda())
    with no_host_sync():
        ms, mp = pose_errors(*args, K, _syms(630))
    assert np.array_equal(ms.cpu().numpy(), bo.pose_errors(pts, _syms(630), gt, est, K)[0])
    for k in (np.array([[np.nan, 1.0, 0, 0]] * 2), np.array([[0.0, 1.0, 0, 0]] * 2), np.ones((3, 4))):
        with pytest.raises(ValueError):
            pose_errors(*args, k, _syms(1))
    with pytest.raises(ValueError):
        pose_errors(args[0][:, :2], *args[1:], K, _syms(1))
    with pytest.raises(ValueError):
        pose_errors(*args, K, np.zeros((0, 3, 4)))
    lib = _lib.load()
    kb = np.array([[np.inf, 1.0, 0.0, 0.0]])
    with pytest.raises(_lib.NopeError):      # the C ABI refuses non-finite intrinsics and bad sizes on its own
        _lib.check(lib.nope_pose_errors(1, 1, 1, 1, 1, 1, kb.ctypes.data, 1, 1, 1, 1, None))
    with pytest.raises(_lib.NopeError):
        _lib.check(lib.nope_pose_errors(1, 0, 1, 1, 1, 1, K.ctypes.data, 1, 1, 1, 1, None))


# ------------------------------------------------------------------ multi-tau VSD
def _frames():
    v, f = ro.sphere(45.0, 2)
    gt = np.stack([ro.look_pose(0.3, 0.2, 0.1, t=(10, -15, 600)), ro.look_pose(-0.2, 0.5, 0.0, t=(-20, 5, 700))])
    preds = np.stack([np.stack([ro.look_pose(0.3 + d, 0.2 - d, 0.1, t=(10 + 10 * i, -15, 600 + 30 * d))
                                for d in (0.0, 0.05, 0.2, 0.6)]) for i in range(2)])
    from nope_b200.vsd import Mesh, render_depth
    m = Mesh(v, f)
    K = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1.0]])
    dg = torch.stack([render_depth(m, gt[i], K, (540, 720))[0] for i in range(2)])
    de = torch.stack([render_depth(m, preds[i], K, (540, 720)) for i in range(2)])
    rng = np.random.default_rng(1)
    dt = dg.double().cpu().numpy() + rng.normal(0, 4.0, dg.shape) * (dg.cpu().numpy() > 0)
    dt[rng.random(dt.shape) < 0.05] = 0
    return torch.from_numpy(np.round(dt * 10) / 10.0).cuda(), dg, de, np.repeat(K4[None], 2, axis=0)


def test_multi_tau_equals_single_tau():
    from nope_b200.vsd import vsd_errors
    dt, dg, de, K = _frames()
    for T in (1, 3, 10, 16):
        taus = np.arange(0.05, 0.51, 0.05)[:T] * 80.0 if T <= 10 else np.linspace(0.5, 60.0, T)
        for cost in ("step", "tlinear"):
            multi = vsd_errors(dt, dg, de, K, tau=taus, cost_type=cost)
            assert multi.shape == (2, 4, T)
            for j, tau in enumerate(taus):
                single = vsd_errors(dt, dg, de, torch.from_numpy(K), tau=float(tau), cost_type=cost)
                assert torch.equal(multi[:, :, j], single), (T, cost, j)
    step = vsd_errors(dt, dg, de, K, tau=[4.0, 20.0, 40.0]).cpu().numpy()
    assert not np.array_equal(step[..., 0], step[..., 2])           # the tolerances do differ


def test_multi_tau_matches_the_reference(golden_dir):
    from nope_b200.vsd import vsd_errors
    from nope_b200.vsd import Mesh, render_depth
    g = dict(np.load(os.path.join(golden_dir, "vsd.npz")))
    F, H, W = g["depth_raw"].shape
    dg, de = [], []
    for i in range(F):                                              # as tests/test_vsd_gpu._golden_inputs
        name = ("box", "sphere")[int(g["mesh_of_frame"][i])]
        m = Mesh(g[f"{name}_vertices"], g[f"{name}_faces"])
        dg.append(render_depth(m, torch.from_numpy(g["gt_poses"][i][None]), g["K"], (H, W))[0])
        de.append(render_depth(m, torch.from_numpy(g["pred_poses"][i]), g["K"], (H, W)))
    dt, dg, de = torch.from_numpy(g["depth_raw"] / 10.0), torch.stack(dg), torch.stack(de)
    K = np.repeat(np.array([[g["K"][0, 0], g["K"][1, 1], g["K"][0, 2], g["K"][1, 2]]]), len(dt), axis=0)
    for s, (delta, tau) in enumerate(g["settings"]):
        out = vsd_errors(dt.cuda(), dg.cuda(), de.cuda(), K, int(delta), [5.0, float(tau), 33.0], "step").cpu().numpy()
        assert np.array_equal(out[..., 1], g["vsd_step"][s])


def test_multi_tau_bad_arguments_and_no_sync():
    from nope_b200 import _lib
    from nope_b200.vsd import vsd_errors
    dt, dg, de, K = _frames()
    with no_host_sync():
        vsd_errors(dt, dg, de, K, tau=[10.0, 20.0])
    for taus in ([], list(range(1, 18)), [1.0, 0.0], [np.nan]):
        with pytest.raises(ValueError):
            vsd_errors(dt, dg, de, K, tau=taus)
    with pytest.raises(ValueError):
        vsd_errors(dt, dg, de, K * [0, 1, 1, 1], tau=[10.0])
    taus, kbad = np.array([10.0, 20.0]), K * [np.nan, 1, 1, 1]
    with pytest.raises(_lib.NopeError):
        _lib.check(_lib.load().nope_vsd_error_taus(1, 1, 1, 2, 4, 8, 8, kbad.ctypes.data, 15.0, 0, taus.ctypes.data,
                                                   2, 1, None))
    with pytest.raises(_lib.NopeError):
        _lib.check(_lib.load().nope_vsd_error_taus(1, 1, 1, 2, 4, 8, 8, K.ctypes.data, 15.0, 0, taus.ctypes.data,
                                                   17, 1, None))


# ------------------------------------------------------------------ eval_bop end to end
def _expected(batch, R, model):
    """the BOP scores from separate render_depth / vsd_errors / pose_errors / average_recall calls"""
    import cv2
    from nope_b200 import bop
    from nope_b200 import vsd as V
    info = model.bop_models[1]
    mesh = model.tless_cad[1]
    B, k = R.shape[:2]
    vsd, mssd, mspd = [], [], []
    for b in range(B):
        poses = np.zeros((1 + k, 4, 4), dtype=np.float32)
        poses[0, :3, :3] = batch["query_pose"][b].numpy()
        poses[1:, :3, :3] = R[b]
        poses[:, :3, 3] = batch["query_translation"][b, :, 0].numpy()
        poses[:, 3, 3] = 1
        d = V.render_depth(mesh, torch.from_numpy(poses), batch["intrinsic"][b], (72, 96))
        dt = torch.from_numpy(cv2.imread(batch["depth_path"][b], -1) / 10.0).cuda()
        vsd.append(V.vsd_errors(dt[None], d[None, 0], d[None, 1:], batch["intrinsic"][b:b + 1],
                                tau=bop.VSD_TAUS * info["diameter"])[0].cpu().numpy())
        t = batch["query_translation"][b:b + 1, :, 0].double()
        ms, mp = bop.pose_errors(mesh.vertices, torch.from_numpy(np.asarray(R[b:b + 1], dtype=np.float64)), t,
                                 batch["query_pose"][b:b + 1].double(), t, batch["intrinsic"][b:b + 1],
                                 info["symmetries"])
        mssd.append(ms[0].cpu().numpy())
        mspd.append(mp[0].cpu().numpy())
    vsd, mssd, mspd = np.stack(vsd), np.stack(mssd), np.stack(mspd)
    out = {}
    for kk in (1, 3, 5):
        if kk <= k:
            for name, value in bop.average_recall(vsd[:, :kk], mssd[:, :kk], mspd[:, :kk], info["diameter"], 96).items():
                out[f"top {kk}, {name}"] = value
    return out, vsd, mssd, mspd


def test_eval_bop_end_to_end(gpu_model, tmp_path, monkeypatch):
    from nope_b200 import bop
    from nope_b200 import vsd as V
    batch, cad, _ = tless_batch(tmp_path, symmetries=FLIPS)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    assert len(model.bop_models[1]["symmetries"]) == 4
    model.logged = {}
    calls = {"render": 0, "vsd": 0, "pose": 0}

    def strict(fn, name):
        def inner(*a, **kw):
            calls[name] += 1
            with no_host_sync():
                return fn(*a, **kw)
        return inner
    monkeypatch.setattr(V, "render_depth", strict(V.render_depth, "render"))
    monkeypatch.setattr(V, "vsd_errors", strict(V.vsd_errors, "vsd"))
    monkeypatch.setattr(bop, "pose_errors", strict(bop.pose_errors, "pose"))
    save = tmp_path / "bop" / "errors.npz"
    out = model.eval_bop(batch, "obj01", save_path=str(save))
    assert calls == {"render": 3, "vsd": 1, "pose": 1}
    monkeypatch.undo()
    _, idx, _ = model.predict_pose(batch["query"], batch["reference"], batch["all_relativeR"], None, k=5)
    R = batch["template_poses"][torch.arange(3)[:, None], idx.cpu()].numpy()
    ref, vsd, mssd, mspd = _expected(batch, R, model)
    assert out == ref
    for key, value in out.items():
        assert model.logged[f"{key}/val_obj01"] == [value]
    assert sorted(out) == sorted(f"top {k}, {n}" for k in (1, 3, 5) for n in ("ar_vsd", "ar_mssd", "ar_mspd", "ar"))
    saved = np.load(str(save))
    assert np.array_equal(saved["vsd"], vsd) and np.array_equal(saved["mssd"], mssd)
    assert np.array_equal(saved["mspd"], mspd) and saved["obj_id"].tolist() == [1, 1, 1]
    # eval_vsd is unchanged by the shared render step: its top-1 VSD is eval_bop's at tau = 20 mm
    vsd20 = model.eval_vsd(batch, "obj01")
    assert vsd20["top 1, vsd_median"] == np.median(V.vsd_errors(
        *_vsd_inputs(batch, R, model), tau=20)[:, 0].cpu().numpy())


def _vsd_inputs(batch, R, model):
    import cv2
    from nope_b200 import vsd as V
    d, dt = [], []
    for b in range(R.shape[0]):
        poses = np.zeros((1 + R.shape[1], 4, 4), dtype=np.float32)
        poses[0, :3, :3] = batch["query_pose"][b].numpy()
        poses[1:, :3, :3] = R[b]
        poses[:, :3, 3] = batch["query_translation"][b, :, 0].numpy()
        poses[:, 3, 3] = 1
        d.append(V.render_depth(model.tless_cad[1], torch.from_numpy(poses), batch["intrinsic"][b], (72, 96)))
        dt.append(torch.from_numpy(cv2.imread(batch["depth_path"][b], -1) / 10.0).cuda())
    d = torch.stack(d)
    return torch.stack(dt), d[:, 0], d[:, 1:], batch["intrinsic"]


def test_eval_bop_with_refined_search(gpu_model, tmp_path):
    from nope_b200.inplane_refine import InplaneRefiner
    batch, cad, _ = tless_batch(tmp_path, symmetries=FLIPS)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    refiner = InplaneRefiner(batch["template_poses"][0], angles=12, steps=2)
    R, *_ = model.predict_pose_inplane_refined(batch["query"], batch["reference"], batch["all_relativeR"], refiner,
                                               k=3)
    out = model.eval_bop(batch, "obj01", R_est=R)
    ref, *_ = _expected(batch, R.detach().cpu().numpy(), model)
    assert out == ref and sorted(out) == sorted(f"top {k}, {n}" for k in (1, 3)
                                                for n in ("ar_vsd", "ar_mssd", "ar_mspd", "ar"))
    with pytest.raises(ValueError):
        model.eval_bop(batch, "obj01", R_est=R[:2])
    model.bop_models.clear()
    with pytest.raises(ValueError):
        model.eval_bop(batch, "obj01")
