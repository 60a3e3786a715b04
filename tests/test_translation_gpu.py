"""GPU: the translation fit (DESIGN.md section 18).  nope_fit_translation_occluded without occluders against the numpy
oracle bit for bit on the same render_depth images after 0 ... 6 updates; the silhouette counts against render_depth's
coverage; accuracy with the true rotation from initial_translation; edge cases (empty mask, a start off screen, batch
composition, no host synchronisation); and eval_bop with t_est."""
import math
import os

import numpy as np
import pytest
import torch

import translation_oracle as to
from _scenes import H, K4, W, inside, make_mesh, render, rot, tless_batch
from _util import no_host_sync

pytestmark = pytest.mark.gpu

def _scene(mesh, seed, F, P, zlo=400.0, zhi=1200.0):
    """F frames: a true pose each (t at zlo ... zhi mm), its mask, and P rotation hypotheses (the first is the true
    one, the others random) -> (R_true [F, 3, 3], t_true [F, 3], masks uint8 [F, H, W] on the GPU, R [F, P, 3, 3])"""
    rng = np.random.default_rng(seed)
    Rt, tt, masks = [], [], []
    while len(Rt) < F:
        R = rot(rng)
        z = rng.uniform(zlo, zhi)
        t = np.array([rng.uniform(-0.2, 0.2) * z, rng.uniform(-0.2, 0.2) * z, z])
        m = render(mesh, R, t) > 0
        if not inside(m):
            continue
        Rt.append(R), tt.append(t), masks.append(m.to(torch.uint8))
    R = np.stack([np.stack([Rt[f]] + [rot(rng) for _ in range(P - 1)]) for f in range(F)])
    return np.stack(Rt), np.stack(tt), torch.stack(masks), R


# ------------------------------------------------------------------ kernel = oracle
@pytest.mark.parametrize("name", ["box", "sphere", "soup"])
@pytest.mark.parametrize("P", [1, 5])
def test_kernel_equals_oracle(name, P):
    """t and iou after 0 ... 6 updates equal the oracle's, which renders with render_depth at its own t; the kernel's
    silhouette counts equal render_depth's coverage at every step"""
    from nope_b200.translation import estimate_translation, initial_translation
    mesh, diameter = make_mesh(name)
    F = 2
    _, _, masks, R = _scene(mesh, 11 + P, F, P)
    K = np.stack([K4 * [1, 1, 1, 1], K4 * [1.0, 1.001, 1.02, 0.98]])
    t0 = initial_translation(masks, K, diameter)
    mh = masks.cpu().numpy()
    for f in range(F):
        assert np.array_equal(t0[f].cpu().numpy(), to.initial_translation(mh[f], K[f], diameter))
    got = [estimate_translation(mesh, R, K, masks, t_init=t0, iters=i, return_stats=True) for i in range(7)]
    got = [tuple(x.cpu().numpy() for x in g) for g in got]
    for f in range(F):
        msk = to.stats(mh[f] != 0)
        for p in range(P):
            t = t0[f].cpu().numpy()
            for i in range(7):
                d = render(mesh, R[f, p], t, K[f]).cpu().numpy()
                sil = to.stats(d > 0, mh[f])
                assert tuple(got[i][2][f, p]) == sil, (f, p, i)
                assert np.array_equal(got[i][0][f, p], t), (f, p, i, got[i][0][f, p], t)
                assert got[i][1][f, p] == to.iou(sil, msk), (f, p, i)
                t = to.update(t, sil, msk, K[f])


def test_workspace_holds_the_final_render():
    """nope_fit_translation_occluded leaves render_depth's image at the returned t in its workspace"""
    from nope_b200 import _lib
    from nope_b200.translation import initial_translation
    from nope_b200.vsd import _stream
    mesh, diameter = make_mesh("sphere")
    _, _, masks, R = _scene(mesh, 3, 2, 3)
    K = np.repeat(K4[None], 2, axis=0)
    t0 = initial_translation(masks, K, diameter)[:, None].expand(2, 3, 3).contiguous()
    Rd = torch.from_numpy(R).cuda().contiguous()
    depth = torch.empty((6, H, W), device="cuda")
    t = torch.empty((2, 3, 3), device="cuda", dtype=torch.float64)
    iou = torch.empty((2, 3), device="cuda", dtype=torch.float64)
    _lib.check(_lib.load().nope_fit_translation_occluded(
        _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
        _lib.ptr(t0), _lib.ptr(masks), None, K.ctypes.data, 2, 3, H, W, 0.05, 3, _lib.ptr(depth), _lib.ptr(t),
        _lib.ptr(iou), None, _stream(torch.device("cuda"))))
    th = t.cpu().numpy()
    for f in range(2):
        for p in range(3):
            assert torch.equal(depth[3 * f + p], render(mesh, R[f, p], th[f, p]))


# ------------------------------------------------------------------ accuracy with the true rotation
@pytest.mark.parametrize("name,box_px,reproj_px", [("box", 2.0, 1.0), ("sphere", 2.0, 1.0), ("soup", 6.0, 6.0)])
def test_accuracy_with_the_true_rotation(name, box_px, reproj_px):
    """32 seeded poses at 400 - 1200 mm, objects inside the frame, masks rendered at the true pose: from
    initial_translation, after the default number of updates, |dz| <= 2 z / sqrt(w h) (two pixels of box size) and
    the origin reprojects within 1 px; from the true translation t stays within 1e-6 mm and the IoU is >= 0.999.
    The triangle soup does not meet the two-pixel bounds: its box ends are sliver tips whose coverage jumps by several
    pixels under a sub-pixel move; it is held to its measured worst case (4.5 box pixels, 5.3 px; DESIGN.md
    section 18) with some room."""
    from nope_b200.translation import DEFAULT_ITERS, estimate_translation
    mesh, diameter = make_mesh(name)
    R_true, t_true, masks, _ = _scene(mesh, 100, 32, 1)
    t, iou = estimate_translation(mesh, R_true, K4, masks, diameter=diameter)
    t, iou = t[:, 0].cpu().numpy(), iou[:, 0].cpu().numpy()
    mh = masks.cpu().numpy()
    for f in range(32):
        n, _, r0, r1, c0, c1 = to.stats(mh[f])
        z = t_true[f, 2]
        assert abs(t[f, 2] - z) <= box_px * z / math.sqrt((c1 - c0 + 1) * (r1 - r0 + 1)), (f, t[f], t_true[f])
        u = K4[:2] * t[f, :2] / t[f, 2] + K4[2:]
        ut = K4[:2] * t_true[f, :2] / z + K4[2:]
        assert np.hypot(*(u - ut)) <= reproj_px, (f, u, ut)
    t, iou = estimate_translation(mesh, R_true, K4, masks, t_init=t_true, iters=DEFAULT_ITERS)
    assert np.abs(t[:, 0].cpu().numpy() - t_true).max() <= 1e-6
    assert iou.min().item() >= 0.999


# ------------------------------------------------------------------ edge cases
def test_empty_mask_and_a_start_off_screen():
    from nope_b200.translation import estimate_translation
    mesh, diameter = make_mesh("box")
    _, t_true, masks, R = _scene(mesh, 7, 3, 2)
    masks[1] = 0
    t_init = np.repeat(t_true[:, None], 2, axis=1)
    t_init[2, 1] = [5000.0, 0.0, 500.0]                           # projects far right of the frame
    t, iou = estimate_translation(mesh, R, K4, masks, t_init=t_init, iters=4)
    t, iou = t.cpu().numpy(), iou.cpu().numpy()
    assert np.isnan(t[1]).all() and np.isnan(iou[1]).all()
    assert np.array_equal(t[2, 1], t_init[2, 1]) and iou[2, 1] == 0.0
    assert np.isfinite(np.delete(t, 1, axis=0)).all() and np.isfinite(np.delete(iou, 1, axis=0)).all()
    t0, _ = estimate_translation(mesh, R, K4, masks, diameter=diameter, iters=2)
    assert np.isnan(t0[1].cpu().numpy()).all()


def test_batch_composition():
    """one frame alone equals the same frame inside a batch, and a hypothesis does not depend on its neighbours"""
    from nope_b200.translation import estimate_translation
    mesh, diameter = make_mesh("sphere")
    _, _, masks, R = _scene(mesh, 21, 4, 5)
    K = np.stack([K4 * [1, 1, 1 + 0.01 * f, 1] for f in range(4)])
    t, iou = estimate_translation(mesh, R, K, masks, diameter=diameter, iters=4)
    for f in range(4):
        a, b = estimate_translation(mesh, R[f:f + 1], K[f:f + 1], masks[f:f + 1], diameter=diameter, iters=4)
        assert torch.equal(a, t[f:f + 1]) and torch.equal(b, iou[f:f + 1])
        for p in (0, 3):
            a, b = estimate_translation(mesh, R[f:f + 1, p], K[f:f + 1], masks[f:f + 1], diameter=diameter, iters=4)
            assert torch.equal(a[:, 0], t[f:f + 1, p]) and torch.equal(b[:, 0], iou[f:f + 1, p])
    perm = [2, 0, 3, 1]
    a, b = estimate_translation(mesh, R[:, perm], K, masks, diameter=diameter, iters=4)
    assert torch.equal(a, t[:, perm]) and torch.equal(b, iou[:, perm])


def test_no_host_synchronisation():
    from nope_b200.translation import estimate_translation, initial_translation
    mesh, diameter = make_mesh("box")
    _, t_true, masks, R = _scene(mesh, 9, 2, 3)
    Rd = torch.from_numpy(R).cuda()
    td = torch.from_numpy(t_true).cuda()
    K = np.repeat(K4[None], 2, axis=0)
    with no_host_sync():
        a = estimate_translation(mesh, Rd, K, masks, diameter=diameter)
        b = estimate_translation(mesh, Rd.float(), K, masks.bool(), t_init=td, iters=2)
        c = initial_translation(masks, K, diameter)
    assert torch.equal(a[0], estimate_translation(mesh, R, K, masks.cpu(), t_init=c.cpu())[0])
    assert b[0].shape == (2, 3, 3) and torch.isfinite(b[0]).all()
    with pytest.raises(ValueError):
        estimate_translation(mesh, R, K, masks)                     # neither t_init nor diameter
    with pytest.raises(ValueError):
        estimate_translation(mesh, R, K, masks[:1], diameter=diameter)
    with pytest.raises(ValueError):
        estimate_translation(mesh, R, K, masks, t_init=td[:, :2], diameter=diameter)
    with pytest.raises(ValueError):
        estimate_translation(mesh, R, K, masks, diameter=diameter, iters=-1)


# ------------------------------------------------------------------ eval_bop with t_est
def test_eval_bop_with_estimated_translation(gpu_model, tmp_path):
    batch, cad, masks = tless_batch(tmp_path)
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.load_models_info(os.path.join(cad, "models_info.json"))
    assert len(model.bop_models[1]["symmetries"]) == 1
    B, k = 3, 2
    R = torch.stack([batch["query_pose"], batch["template_poses"][:, 5]], dim=1)      # the truth, a wrong view
    t_gt = batch["query_translation"][:, None, :, 0].expand(B, k, 3).double()
    # t_est at the true translation: exactly eval_bop's scores without it
    ref_path, gt_path = tmp_path / "ref.npz", tmp_path / "gt.npz"
    ref = model.eval_bop(batch, "obj01", R_est=R, save_path=str(ref_path))
    same = model.eval_bop(batch, "obj01", R_est=R, save_path=str(gt_path), t_est=t_gt)
    assert same == ref
    a, b = np.load(str(ref_path)), np.load(str(gt_path))
    assert all(np.array_equal(a[key], b[key]) for key in ("vsd", "mssd", "mspd"))
    # t_est from the masks: MSSD of the true rotation is |t_est - t_gt|
    t_est, iou = model.estimate_translation(batch, R, masks)
    assert t_est.shape == (B, k, 3) and iou.shape == (B, k) and (iou[:, 0] > 0.8).all()
    t_est[2, 1] = t_gt[2, 1].to(t_est.device)                                       # one row keeps the truth
    est_path = tmp_path / "est.npz"
    model.eval_bop(batch, "obj01", R_est=R, save_path=str(est_path), t_est=t_est)
    c = np.load(str(est_path))
    dt = np.linalg.norm(t_est.cpu().numpy() - t_gt.numpy(), axis=2)
    assert np.abs(c["mssd"][:, 0] - dt[:, 0]).max() <= 1e-9 * np.abs(t_gt.numpy()).max(), (c["mssd"], dt)
    assert (dt[:, 0] > 0).any()                                                        # t_est is used
    assert np.array_equal(c["vsd"][2, 1], a["vsd"][2, 1]) and c["mssd"][2, 1] == a["mssd"][2, 1]
    with pytest.raises(ValueError):
        model.eval_bop(batch, "obj01", R_est=R, t_est=t_est[:, :1])
