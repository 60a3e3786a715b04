"""GPU: the contour refinement (DESIGN.md section 20).  nope_mask_sdf against the numpy oracle bit for bit, at 720 x 540
and on edge cases; nope_refine_contour_occluded without occluders against the oracle bit for bit, integer sums included,
on the same render_depth images after 0 ... 6 updates; the true pose kept to the bit; accuracy from perturbed starts;
batch independence; masks without a contour; no host synchronisation; `PoseConditional.refine_contour` with rerank, and
eval_bop at refined poses."""
import os

import numpy as np
import pytest
import torch

import contour_refine_oracle as cro
from _scenes import H, K4, W, angle, make_mesh, perturb, render, rot, scene, tless_batch
from _util import no_host_sync

pytestmark = pytest.mark.gpu

TAUS = np.geomspace(0.15, 0.02, 7)


def _masks_scene(mesh, seed, F, P, K=None, deg=5.0, mm=10.0):
    """(R_true, t_true, masks uint8 [F, H, W] on the GPU = the render at the true pose, R0, t0)"""
    R_true, t_true, _, M, R0, t0 = scene(mesh, seed, F, P, K=K, sensor=False, background=False, deg=deg, mm=mm)
    return R_true, t_true, M, R0, t0


# ------------------------------------------------------------------ the signed distance field
def test_mask_sdf_equals_oracle():
    from nope_b200.contour_refine import mask_sdf
    mesh, _ = make_mesh("box")
    _, _, M, _, _ = _masks_scene(mesh, 5, 2, 1)
    got = mask_sdf(M).cpu().numpy()
    for f in range(2):
        assert np.array_equal(got[f], cro.sdf(M[f].cpu().numpy()))
    rng = np.random.default_rng(1)
    cases = [rng.random((37, 53)) < p for p in (0.02, 0.3, 0.97)]
    m = np.zeros((37, 53), bool)
    m[:5, :9] = m[30:, 40:] = True                            # touching the frame border
    cases.append(m)
    m = np.zeros((37, 53), bool)
    m[20, 7] = True                                           # one pixel
    cases += [m, np.zeros((37, 53), bool), np.ones((37, 53), bool)]
    got = mask_sdf(torch.from_numpy(np.stack(cases))).cpu().numpy()      # host masks go to the current device
    for f, m in enumerate(cases):
        assert np.array_equal(got[f], cro.sdf(m), equal_nan=True), f
    assert np.isnan(got[-2:]).all()
    one = mask_sdf(np.ones((1, 1), np.uint8))
    assert one.shape == (1, 1, 1) and torch.isnan(one).all()
    line = np.zeros((1, 9), bool)
    line[0, 2] = True
    assert np.array_equal(mask_sdf(line)[0].cpu().numpy(), cro.sdf(line))


# ------------------------------------------------------------------ kernel = oracle
@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
@pytest.mark.parametrize("P", [1, 5])
def test_kernel_equals_oracle(name, P):
    """R, t, the fit and the integer sums after 0 ... 6 updates equal the oracle's, which renders with render_depth at
    its own pose; frame 1 has a perturbed K"""
    from nope_b200.contour_refine import refine_pose_contour
    mesh, _ = make_mesh(name)
    F = 2
    K = np.stack([K4, K4 * [1.0, 1.001, 1.02, 0.98]])
    _, _, M, R0, t0 = _masks_scene(mesh, 41 + P, F, P, K=K)
    got = [refine_pose_contour(mesh, R0, t0, K, M, iters=i, tau=TAUS[:i + 1], return_sums=True) for i in range(7)]
    got = [(g[0].cpu().numpy(), g[1].cpu().numpy(), torch.stack([g[2][k] for k in ("n_in", "n_contour", "rms",
           "iou")], -1).cpu().numpy(), g[3].cpu().numpy()) for g in got]
    Mh = M.cpu().numpy()
    rho = mesh.radius
    for f in range(F):
        phi, s = cro.sdf(Mh[f]), cro.box_size(Mh[f])
        for p in range(P):
            R, t = R0[f, p], t0[f, p]
            for i in range(7):
                D = render(mesh, R, t, K[f]).cpu().numpy()
                tau = TAUS[i] * s
                sums, nc = cro.accumulate(D, phi, K[f], t, tau, rho)
                assert np.array_equal(got[i][3][f, p], sums), (f, p, i, got[i][3][f, p] - sums)
                assert np.array_equal(got[i][0][f, p], R) and np.array_equal(got[i][1][f, p], t), (f, p, i)
                nin = float(sums[-1])
                with np.errstate(invalid="ignore", divide="ignore"):
                    rms = tau * np.sqrt(np.float64(cro.dro.unfix(sums[-2])) / np.float64(nin))
                fit = np.array([nin, float(nc), rms, cro.iou(D, Mh[f])])
                assert np.array_equal(got[i][2][f, p], fit, equal_nan=True), (f, p, i, got[i][2][f, p], fit)
                R, t = cro.solve(sums, R, t, tau, K[f], rho)
            assert got[6][3][f, p, -1] > 50                               # pairs were found


def test_workspace_holds_the_final_render():
    from nope_b200 import _lib
    from nope_b200.vsd import _stream
    mesh, _ = make_mesh("sphere")
    _, _, M, R0, t0 = _masks_scene(mesh, 3, 2, 3)
    K = np.repeat(K4[None], 2, axis=0)
    Rd, td = torch.from_numpy(R0).cuda().contiguous(), torch.from_numpy(t0).cuda().contiguous()
    depth = torch.empty((6, H, W), device="cuda")
    R = torch.empty((2, 3, 3, 3), device="cuda", dtype=torch.float64)
    t = torch.empty((2, 3, 3), device="cuda", dtype=torch.float64)
    fit = torch.empty((2, 3, 4), device="cuda", dtype=torch.float64)
    tau = TAUS[:4].copy()
    _lib.check(_lib.load().nope_refine_contour_occluded(
        _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
        _lib.ptr(td), _lib.ptr(M), None, K.ctypes.data, 2, 3, H, W, mesh.radius, tau.ctypes.data, 3, 0.05,
        _lib.ptr(depth), _lib.ptr(R), _lib.ptr(t), _lib.ptr(fit), None, _stream(torch.device("cuda"))))
    Rh, th = R.cpu().numpy(), t.cpu().numpy()
    for f in range(2):
        for p in range(3):
            assert torch.equal(depth[3 * f + p], render(mesh, Rh[f, p], th[f, p]))


@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
def test_the_true_pose_stays_to_the_bit(name):
    from nope_b200.contour_refine import refine_pose_contour
    mesh, _ = make_mesh(name)
    R_true, t_true, M, _, _ = _masks_scene(mesh, 7, 4, 1)
    R, t, fit, sums = refine_pose_contour(mesh, R_true, t_true, K4, M, return_sums=True)
    assert np.array_equal(R[:, 0].cpu().numpy(), R_true) and np.array_equal(t[:, 0].cpu().numpy(), t_true)
    assert (fit["rms"] == 0).all() and (fit["iou"] == 1).all() and (fit["n_in"] > 50).all()
    assert (sums[..., 21:28] == 0).all()


# ------------------------------------------------------------------ accuracy
# (median rotation error deg, median translation error mm, smallest IoU) after the default schedule, rotations 2.5 -
# 5 deg off, translations 5 - 10 mm off ("offset", median 4.1 deg / 8.5 mm) or from estimate_translation at the
# perturbed rotation ("box fit", 4.1 deg / 9.1 mm on the box), the mask the render at the true pose.  Measured (DESIGN.md
# section 20): box 0.44 deg / 1.5 mm and 0.98 deg / 3.3 mm, icosphere 0.40 mm from both starts, soup 0.17 deg / 4.4 mm
# and 0.08 deg / 2.4 mm; the bounds give them room.  The box must also halve both median errors from either start.
# The sphere's rotation is unobservable from its silhouette and is not held.
BOUNDS = {("box", "offset"): (1.0, 3.0, 0.95), ("box", "box fit"): (1.5, 4.5, 0.9),
          ("sphere", "offset"): (None, 1.0, 0.95), ("sphere", "box fit"): (None, 1.0, 0.95),
          ("soup", "offset"): (0.5, 7.0, 0.6), ("soup", "box fit"): (0.5, 4.0, 0.9)}


@pytest.mark.parametrize("start", ["offset", "box fit"])
@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
def test_accuracy_from_perturbed_starts(name, start):
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import estimate_translation
    mesh, diameter = make_mesh(name)
    R_true, t_true, M, R0, t0 = _masks_scene(mesh, 100, 16, 1)
    if start == "box fit":
        t0 = estimate_translation(mesh, R0, K4, M, diameter=diameter)[0].cpu().numpy()
    R, t, fit = refine_pose_contour(mesh, R0, t0, K4, M)
    R, t = R[:, 0].cpu().numpy(), t[:, 0].cpu().numpy()
    deg, mm, iou = BOUNDS[name, start]
    err_t = np.linalg.norm(t - t_true, axis=1)
    err_t0 = np.linalg.norm(t0[:, 0] - t_true, axis=1)
    err_r = np.array([angle(R[f], R_true[f]) for f in range(16)])
    err_r0 = np.array([angle(R0[f, 0], R_true[f]) for f in range(16)])
    assert np.median(err_t) <= mm, (err_t, err_t0)
    assert deg is None or np.median(err_r) <= deg, (err_r, err_r0)
    if name == "box":
        assert np.median(err_t) <= 0.5 * np.median(err_t0) and np.median(err_r) <= 0.5 * np.median(err_r0)
    assert (fit["iou"] > iou).all(), fit["iou"]


# ------------------------------------------------------------------ batch independence and edge cases
def test_batch_independence():
    from nope_b200.contour_refine import refine_pose_contour
    mesh, _ = make_mesh("box")
    K = np.stack([K4 * [1, 1, 1 + 0.01 * f, 1] for f in range(3)])
    _, _, M, R0, t0 = _masks_scene(mesh, 21, 3, 4, K=K)
    R, t, fit = refine_pose_contour(mesh, R0, t0, K, M)
    for f in range(3):
        a, b, c = refine_pose_contour(mesh, R0[f:f + 1], t0[f:f + 1], K[f:f + 1], M[f:f + 1])
        assert torch.equal(a, R[f:f + 1]) and torch.equal(b, t[f:f + 1])
        assert all(torch.equal(c[k], fit[k][f:f + 1]) for k in c)
        for p in (0, 3):
            a, b, c = refine_pose_contour(mesh, R0[f:f + 1, p], t0[f:f + 1, p], K[f:f + 1], M[f:f + 1])
            assert torch.equal(a[:, 0], R[f:f + 1, p]) and torch.equal(b[:, 0], t[f:f + 1, p])
            assert all(torch.equal(c[k][:, 0], fit[k][f:f + 1, p]) for k in c)
    perm = [2, 0, 3, 1]
    a, b, c = refine_pose_contour(mesh, R0[:, perm], t0[:, perm], K, M)
    assert torch.equal(a, R[:, perm]) and torch.equal(b, t[:, perm])
    assert all(torch.equal(c[k], fit[k][:, perm]) for k in c)


def test_empty_and_full_masks_keep_the_pose():
    from nope_b200.contour_refine import refine_pose_contour
    mesh, _ = make_mesh("box")
    _, _, M, R0, t0 = _masks_scene(mesh, 8, 3, 2)
    M[1] = 0
    M[2] = 1
    R, t, fit = refine_pose_contour(mesh, R0, t0, K4, M)
    R, t = R.cpu().numpy(), t.cpu().numpy()
    for f in (1, 2):
        assert np.array_equal(R[f], R0[f]) and np.array_equal(t[f], t0[f])
        assert (fit["n_in"][f] == 0).all() and (fit["n_contour"][f] > 0).all()
        assert fit["rms"][f].isnan().all() and fit["iou"][f].isnan().all()
    assert torch.isfinite(fit["iou"][0]).all() and not np.array_equal(t[0], t0[0])


def test_no_host_synchronisation():
    from nope_b200.contour_refine import mask_sdf, refine_pose_contour
    mesh, _ = make_mesh("box")
    _, _, M, R0, t0 = _masks_scene(mesh, 9, 2, 3)
    Rd, td = torch.from_numpy(R0).cuda(), torch.from_numpy(t0).cuda()
    K = np.repeat(K4[None], 2, axis=0)
    with no_host_sync():
        a = refine_pose_contour(mesh, Rd, td, K, M)
        b = refine_pose_contour(mesh, Rd.float(), td[:, 0], K, M.bool(), iters=2, tau=0.05)
        s = mask_sdf(M)
    c = refine_pose_contour(mesh, R0, t0, K, M.cpu())
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert b[0].shape == (2, 3, 3, 3) and torch.isfinite(b[1]).all()
    assert s.shape == M.shape


# ------------------------------------------------------------------ PoseConditional.refine_contour and eval_bop
def test_rerank_puts_the_true_rotation_first(gpu_model, tmp_path):
    batch, cad, masks = tless_batch(tmp_path)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    B, k = 3, 5
    rng = np.random.default_rng(4)
    R_gt = batch["query_pose"].double().numpy()
    R = np.stack([np.stack([rot(rng) for _ in range(k)]) for _ in range(B)])
    for b in range(B):
        R[b, 3] = R_gt[b]
    t = batch["query_translation"][:, None, :, 0].expand(B, k, 3).double()
    R1, t1, iou = model.refine_contour(batch, R, t, masks)
    assert R1.shape == (B, k, 3, 3) and t1.shape == (B, k, 3) and iou.shape == (B, k)
    R2, t2, iou2 = model.refine_contour(batch, R, t, masks, rerank=True)
    order = torch.sort(-iou, dim=1, stable=True).indices
    rows = torch.arange(B, device=order.device)[:, None]
    assert torch.equal(R2, R1[rows, order]) and torch.equal(t2, t1[rows, order]) and torch.equal(iou2, iou[rows, order])
    assert (order[:, 0] == 3).all(), iou
    assert (iou2[:, :-1] >= iou2[:, 1:]).all()


def test_eval_bop_at_refined_poses(gpu_model, tmp_path):
    """the median MSSD at poses refined from perturbed starts is lower than at the starts"""
    batch, cad, masks = tless_batch(tmp_path)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    B, k = 3, 4
    rng = np.random.default_rng(6)
    R_gt = batch["query_pose"].double().numpy()
    t_gt = batch["query_translation"][:, :, 0].double().numpy()
    starts = [[perturb(rng, R_gt[b], t_gt[b], 4.0, 6.0) for _ in range(k)] for b in range(B)]
    R0 = np.stack([np.stack([s[0] for s in row]) for row in starts])
    t0 = np.stack([np.stack([s[1] for s in row]) for row in starts])
    p0, p1 = tmp_path / "start.npz", tmp_path / "refined.npz"
    model.eval_bop(batch, "obj01", R_est=R0, t_est=t0, save_path=str(p0))
    R1, t1, _ = model.refine_contour(batch, R0, t0, masks)
    model.eval_bop(batch, "obj01", R_est=R1, t_est=t1, save_path=str(p1))
    a, b = np.load(str(p0)), np.load(str(p1))
    assert np.median(b["mssd"]) < np.median(a["mssd"]), (a["mssd"], b["mssd"])
