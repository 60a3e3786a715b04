"""GPU: the depth refinement (DESIGN.md section 19).  nope_refine_depth against the numpy oracle bit for bit, integer
sums included, on the same render_depth images after 0 ... 6 updates; accuracy from perturbed starts on sensor-like
depth (quantised to 0.1 mm, seeded noise and holes, a background plane behind the object); the true pose kept;
batch independence; edge cases; no host synchronisation; `PoseConditional.refine_depth` with rerank, and eval_bop
at refined poses."""
import os

import numpy as np
import pytest
import torch

import depth_refine_oracle as dro
from _scenes import H, K4, W, angle, make_mesh, perturb, render, rot, scene, tless_batch
from _util import no_host_sync

pytestmark = pytest.mark.gpu

TAUS = np.geomspace(20.0, 2.0, 7)


# ------------------------------------------------------------------ kernel = oracle
@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
@pytest.mark.parametrize("P", [1, 5])
def test_kernel_equals_oracle(name, P):
    """R, t, the fit and the integer sums after 0 ... 6 updates equal the oracle's, which renders with render_depth at
    its own pose; frame 1 has a perturbed K; the P = 5 case uses masks"""
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh(name)
    F = 2
    K = np.stack([K4, K4 * [1.0, 1.001, 1.02, 0.98]])
    _, _, S, M, R0, t0 = scene(mesh, 31 + P, F, P, K=K)
    masks = M if P == 5 else None
    got = [refine_pose_depth(mesh, R0, t0, K, S, masks=masks, iters=i, tau=TAUS[:i + 1], return_sums=True)
           for i in range(7)]
    got = [(g[0].cpu().numpy(), g[1].cpu().numpy(), torch.stack([g[2][k] for k in ("n_in", "n_valid", "rms",
           "score")], -1).cpu().numpy(), g[3].cpu().numpy()) for g in got]
    Sh = S.cpu().numpy()
    Mh = None if masks is None else masks.cpu().numpy()
    rho = mesh.radius
    for f in range(F):
        nv = dro.valid_count(Sh[f], None if Mh is None else Mh[f])
        for p in range(P):
            R, t = R0[f, p], t0[f, p]
            for i in range(7):
                sums = dro.accumulate(render(mesh, R, t, K[f]).cpu().numpy(), Sh[f], None if Mh is None else Mh[f],
                                      K[f], t, TAUS[i], rho)
                assert np.array_equal(got[i][3][f, p], sums), (f, p, i, got[i][3][f, p] - sums)
                assert np.array_equal(got[i][0][f, p], R) and np.array_equal(got[i][1][f, p], t), (f, p, i)
                assert np.array_equal(got[i][2][f, p], dro.fit_stats(sums, nv, TAUS[i]), equal_nan=True), (f, p, i)
                R, t = dro.solve(sums, R, t, TAUS[i], rho)
            assert got[6][3][f, p, -1] > 100                              # pairs were found


def test_workspace_holds_the_final_render():
    from nope_b200 import _lib
    from nope_b200.vsd import _stream
    mesh, _ = make_mesh("sphere")
    _, _, S, _, R0, t0 = scene(mesh, 3, 2, 3)
    K = np.repeat(K4[None], 2, axis=0)
    Rd, td = torch.from_numpy(R0).cuda().contiguous(), torch.from_numpy(t0).cuda().contiguous()
    depth = torch.empty((6, H, W), device="cuda")
    R = torch.empty((2, 3, 3, 3), device="cuda", dtype=torch.float64)
    t = torch.empty((2, 3, 3), device="cuda", dtype=torch.float64)
    fit = torch.empty((2, 3, 4), device="cuda", dtype=torch.float64)
    tau = TAUS[:4].copy()
    _lib.check(_lib.load().nope_refine_depth(
        _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
        _lib.ptr(td), _lib.ptr(S), None, K.ctypes.data, 2, 3, H, W, mesh.radius, tau.ctypes.data, 3, 0.05,
        _lib.ptr(depth), _lib.ptr(R), _lib.ptr(t), _lib.ptr(fit), None, _stream(torch.device("cuda"))))
    Rh, th = R.cpu().numpy(), t.cpu().numpy()
    for f in range(2):
        for p in range(3):
            assert torch.equal(depth[3 * f + p], render(mesh, Rh[f, p], th[f, p]))


# ------------------------------------------------------------------ accuracy
# (median rotation error deg, median translation error mm) after the default schedule, and the most any hypothesis
# may end up further from the truth than it started (deg, mm): from the measured table of DESIGN.md section 19 (16
# frames per mesh, 720 x 540, starts 2.5 - 5 deg and 5 - 10 mm off), with room.  Projective point-to-plane ICP cannot
# see a slide along a large flat face whose edges pair with other faces, so some box and soup starts keep part of
# their offset; none may get worse.  The sphere's rotation is unobservable: it is only held not to drift.  The soup
# of unconnected triangles has depth normals across gaps between triangles, and some of its starts wander off
# (measured: up to 2.8 mm and 29 deg worse than the start); it is held to that measured level.
BOUNDS = {"box": (0.2, 0.5, 0.5, 1.0), "sphere": (None, 0.1, 1.0, 0.1), "soup": (1.5, 1.0, 40.0, 4.0)}


@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
def test_accuracy_from_perturbed_starts(name):
    """sensor-like depth with a background plane, the mask, the default schedule"""
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh(name)
    R_true, t_true, S, M, R0, t0 = scene(mesh, 100, 16, 1)
    R, t, fit = refine_pose_depth(mesh, R0, t0, K4, S, masks=M)
    R, t = R[:, 0].cpu().numpy(), t[:, 0].cpu().numpy()
    deg, mm, worse_deg, worse_mm = BOUNDS[name]
    err_t = np.linalg.norm(t - t_true, axis=1)
    err_t0 = np.linalg.norm(t0[:, 0] - t_true, axis=1)
    err_r = np.array([angle(R[f], R_true[f]) for f in range(16)])
    err_r0 = np.array([angle(R0[f, 0], R_true[f]) for f in range(16)])
    assert np.median(err_t) <= mm and (err_t <= err_t0 + worse_mm).all(), (err_t, err_t0)
    assert deg is None or np.median(err_r) <= deg, err_r
    assert (err_r <= err_r0 + worse_deg).all(), (err_r, err_r0)
    assert (fit["n_in"] > 100).all()


@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
def test_the_true_pose_stays(name):
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh(name)
    R_true, t_true, S, _, _, _ = scene(mesh, 7, 4, 1, sensor=False, background=False)
    R, t, fit = refine_pose_depth(mesh, R_true, t_true, K4, S)
    R, t = R[:, 0].cpu().numpy(), t[:, 0].cpu().numpy()
    assert np.abs(t - t_true).max() <= 1e-6
    assert max(angle(R[f], R_true[f]) for f in range(4)) <= 1e-6
    assert (fit["rms"] == 0).all()


def test_the_mask_keeps_the_background_out():
    """a background plane 40 mm behind the box, within the first tolerances: with the mask the fit is bit for bit the
    fit without a background; without the mask the plane's pixels count as valid"""
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh("box")
    R_true, t_true, S, M, R0, t0 = scene(mesh, 55, 8, 1)
    R_true2, t_true2, S2, M2, _, _ = scene(mesh, 55, 8, 1, background=False)
    R, t, fit = refine_pose_depth(mesh, R0, t0, K4, S, masks=M)
    R2, t2, fit2 = refine_pose_depth(mesh, R0, t0, K4, S2, masks=M2)
    assert torch.equal(R, R2) and torch.equal(t, t2)                  # the mask hides the plane entirely
    assert np.median(np.linalg.norm(t[:, 0].cpu().numpy() - t_true, axis=1)) <= BOUNDS["box"][1]
    _, _, fit3 = refine_pose_depth(mesh, R0, t0, K4, S)
    assert (fit3["n_valid"] > fit["n_valid"]).all()                     # without a mask the plane counts as valid


# ------------------------------------------------------------------ batch independence and edge cases
def test_batch_independence():
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh("sphere")
    K = np.stack([K4 * [1, 1, 1 + 0.01 * f, 1] for f in range(3)])
    _, _, S, M, R0, t0 = scene(mesh, 21, 3, 4, K=K)
    R, t, fit = refine_pose_depth(mesh, R0, t0, K, S, masks=M)
    for f in range(3):
        a, b, c = refine_pose_depth(mesh, R0[f:f + 1], t0[f:f + 1], K[f:f + 1], S[f:f + 1], masks=M[f:f + 1])
        assert torch.equal(a, R[f:f + 1]) and torch.equal(b, t[f:f + 1])
        assert all(torch.equal(c[k], fit[k][f:f + 1]) for k in c)
        for p in (0, 3):
            a, b, c = refine_pose_depth(mesh, R0[f:f + 1, p], t0[f:f + 1, p], K[f:f + 1], S[f:f + 1],
                                        masks=M[f:f + 1])
            assert torch.equal(a[:, 0], R[f:f + 1, p]) and torch.equal(b[:, 0], t[f:f + 1, p])
            assert torch.equal(c["score"][:, 0], fit["score"][f:f + 1, p])
    perm = [2, 0, 3, 1]
    a, b, c = refine_pose_depth(mesh, R0[:, perm], t0[:, perm], K, S, masks=M)
    assert torch.equal(a, R[:, perm]) and torch.equal(b, t[:, perm]) and torch.equal(c["rms"], fit["rms"][:, perm])


def test_empty_mask_or_depth_keeps_the_pose():
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh("box")
    _, _, S, M, R0, t0 = scene(mesh, 8, 3, 2)
    M[1] = 0
    S[2] = 0
    R, t, fit = refine_pose_depth(mesh, R0, t0, K4, S, masks=M)
    R, t = R.cpu().numpy(), t.cpu().numpy()
    for f in (1, 2):
        assert np.array_equal(R[f], R0[f]) and np.array_equal(t[f], t0[f])
        assert (fit["n_in"][f] == 0).all() and (fit["n_valid"][f] == 0).all()
        assert fit["rms"][f].isnan().all() and fit["score"][f].isnan().all()
    assert torch.isfinite(fit["score"][0]).all() and not np.array_equal(t[0], t0[0])


def test_no_host_synchronisation():
    from nope_b200.depth_refine import refine_pose_depth
    mesh, _ = make_mesh("box")
    _, _, S, M, R0, t0 = scene(mesh, 9, 2, 3)
    Rd, td = torch.from_numpy(R0).cuda(), torch.from_numpy(t0).cuda()
    K = np.repeat(K4[None], 2, axis=0)
    with no_host_sync():
        a = refine_pose_depth(mesh, Rd, td, K, S, masks=M)
        b = refine_pose_depth(mesh, Rd.float(), td[:, 0], K, S.float(), masks=M.bool(), iters=2, tau=5.0)
    c = refine_pose_depth(mesh, R0, t0, K, S.cpu(), masks=M.cpu())
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert b[0].shape == (2, 3, 3, 3) and torch.isfinite(b[1]).all()


# ------------------------------------------------------------------ PoseConditional.refine_depth and eval_bop
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
    R1, t1, score = model.refine_depth(batch, R, t, masks=masks)
    assert R1.shape == (B, k, 3, 3) and t1.shape == (B, k, 3) and score.shape == (B, k)
    R2, t2, score2 = model.refine_depth(batch, R, t, masks=masks, rerank=True)
    order = torch.sort(-score, dim=1, stable=True).indices
    rows = torch.arange(B, device=order.device)[:, None]
    assert torch.equal(R2, R1[rows, order]) and torch.equal(score2, score[rows, order])
    assert (order[:, 0] == 3).all(), score
    assert (score2[:, :-1] >= score2[:, 1:]).all()


def test_eval_bop_at_refined_poses(gpu_model, tmp_path):
    """MSSD at poses refined from perturbed starts is no worse than at the starts, row by row; refined from the truth,
    eval_bop gives the unrefined scores"""
    batch, cad, masks = tless_batch(tmp_path)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    B = 3
    rng = np.random.default_rng(6)
    R_gt = batch["query_pose"].double().numpy()
    t_gt = batch["query_translation"][:, :, 0].double().numpy()
    R0, t0 = zip(*[perturb(rng, R_gt[b], t_gt[b], 3.0, 4.0) for b in range(B)])
    R0, t0 = np.stack(R0)[:, None], np.stack(t0)[:, None]
    p0, p1 = tmp_path / "start.npz", tmp_path / "refined.npz"
    model.eval_bop(batch, "obj01", R_est=R0, t_est=t0, save_path=str(p0))
    R1, t1, _ = model.refine_depth(batch, R0, t0, masks=masks)
    model.eval_bop(batch, "obj01", R_est=R1, t_est=t1, save_path=str(p1))
    a, b = np.load(str(p0)), np.load(str(p1))
    assert (b["mssd"] <= a["mssd"]).all(), (a["mssd"], b["mssd"])
    # from the truth: the pose moves by at most the sensor noise's pull, and the scores stay
    tg = torch.from_numpy(t_gt)[:, None]
    ref = model.eval_bop(batch, "obj01", R_est=R_gt[:, None], t_est=tg)
    R2, t2, _ = model.refine_depth(batch, R_gt[:, None], tg, masks=masks)
    assert (t2.cpu() - tg).abs().max() <= 1.0
    assert model.eval_bop(batch, "obj01", R_est=R2, t_est=t2) == ref
