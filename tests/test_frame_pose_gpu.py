"""GPU: the crop camera and predict_pose_frames (DESIGN.md section 23).  crop_camera_kernel and crop_rotate_kernel
against the numpy oracle bit for bit; the crop camera against the rasterizer (a frame render warped by frame_crops
against a render in the crop camera); predict_pose_frames with the search stubbed to the truth, and with the seeded
engine against the hand-written chain of its stages; shared frames; host synchronisation.  The weights are seeded:
nothing here says how accurate a trained model is on real frames."""
import math
import types

import numpy as np
import pytest
import torch

import crop_camera_oracle as cco
from _scenes import H, K3, W, inside, make_mesh, pose, rot, with_objects
from _util import count_host_syncs, same_bits

pytestmark = pytest.mark.gpu

S = 256
def _scene(mesh, seed, n, corners=False):
    """n true poses with the object wholly inside the 720 x 540 frame, its centre anywhere in the frame (or within
    110 px of a frame corner), 400 ... 1200 mm deep -> (R [n, 3, 3], t [n, 3], masks uint8 0 / 255 [n, H, W] CUDA)"""
    from nope_b200.vsd import render_depth
    rng = np.random.default_rng(seed)
    Rs, ts, ms = [], [], []
    while len(Rs) < n:
        R = rot(rng)
        z = rng.uniform(700.0 if corners else 400.0, 1200.0)
        if corners:
            cu, cv = [(0, 0), (W, 0), (0, H), (W, H)][len(Rs) % 4]
            u, v = abs(cu - rng.uniform(60, 110)), abs(cv - rng.uniform(60, 110))
        else:
            u, v = rng.uniform(0, W), rng.uniform(0, H)
        t = np.linalg.solve(K3, [u, v, 1.0]) * z
        m = render_depth(mesh, torch.from_numpy(pose(R, t)), K3, (H, W))[0] > 0
        if not inside(m):
            continue
        Rs.append(R), ts.append(t), ms.append(m.to(torch.uint8) * 255)
    return np.stack(Rs), np.stack(ts), torch.stack(ms)


def _frames(masks):
    """uint8 RGB frames: white object on black"""
    return masks[..., None].expand(*masks.shape, 3).contiguous()


# ------------------------------------------------------------------ kernels = oracle
@pytest.mark.parametrize("keep_inplane", [True, False])
@pytest.mark.parametrize("F", [1, 7, 300])
def test_crop_camera_and_rotate_equal_the_oracle(keep_inplane, F):
    from nope_b200.crop import crop_camera, to_camera, to_crop
    P = cco.seeded_poses(F + keep_inplane, F, keep_inplane, K3)
    if not keep_inplane:
        P[:, :3, 3] /= 1000.0
    if F == 7:
        P[0, :3, 3] = [0.0, 0.0, 0.7]                        # on the axis
        if not keep_inplane:
            P[0, :3, :3] = np.eye(3)                          # and crop_frame's image-axes fallback
    Rv = crop_camera(torch.from_numpy(P).cuda(), keep_inplane)
    Rv_o = cco.crop_camera(P, keep_inplane)
    assert Rv.dtype == torch.float64 and Rv.shape == (F, 3, 3) and Rv.is_cuda
    assert same_bits(Rv, Rv_o)
    if F == 7:
        assert torch.equal(Rv[0].cpu(), torch.eye(3, dtype=torch.float64))
    assert same_bits(crop_camera(torch.from_numpy(P[0]).cuda(), keep_inplane), Rv_o[0])
    g = torch.Generator().manual_seed(F)
    for Pn in (1, 5, 36):
        Q, _ = torch.linalg.qr(torch.randn(F, Pn, 3, 3, generator=g, dtype=torch.float64))
        for dtype in (torch.float64, torch.float32):
            R = Q.to(dtype).cuda()
            for fn, to_cam in ((to_camera, True), (to_crop, False)):
                got = fn(R, Rv)
                assert got.dtype == torch.float64 and got.shape == R.shape
                assert same_bits(got, cco.crop_rotate(Rv_o, R.double().cpu().numpy(), to_cam))
    # [F, 3, 3] input; out aliasing R through the C ABI
    assert same_bits(to_camera(Q[:, 0].cuda(), Rv), cco.crop_rotate(Rv_o, Q[:, :1].numpy(), True)[:, 0])
    from nope_b200 import _lib
    for to_cam in (1, 0):
        R = Q.cuda().contiguous()
        _lib.check(_lib.load().nope_crop_rotate(_lib.ptr(Rv), F, _lib.ptr(R), 36, to_cam, _lib.ptr(R), None))
        assert same_bits(R, cco.crop_rotate(Rv_o, Q.numpy(), bool(to_cam)))


def test_round_trip_and_non_finite_rotations():
    from nope_b200.crop import crop_camera, to_camera, to_crop
    P = cco.seeded_poses(3, 50, True, K3)
    Rv = crop_camera(torch.from_numpy(P).cuda())
    Q, _ = torch.linalg.qr(torch.randn(50, 4, 3, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64))
    R = Q.cuda()
    assert (to_camera(to_crop(R, Rv), Rv) - R).abs().max() <= 1e-15
    R[3, 2, 1, 1] = float("nan")
    out = to_camera(R, Rv)
    assert out[3, 2, :, 1].isnan().all() and not out[3, 2, :, 0].isnan().any() and not out[:3].isnan().any()


def test_python_refusals_on_the_device():
    from nope_b200.crop import crop_camera, to_camera
    good = torch.from_numpy(cco.seeded_poses(0, 3, True, K3)).cuda()
    for bad in (good.clone().fill_(float("nan")), torch.cat([good[:2], -good[2:]]), good[:, :3]):
        with pytest.raises(ValueError):
            crop_camera(bad)
    Rv = crop_camera(good)
    R = torch.eye(3, device="cuda").repeat(3, 2, 1, 1)
    for args in ((R.half(), Rv), (R, Rv.float()), (R[:2], Rv), (R[..., :2], Rv), (R[:, :0], Rv)):
        with pytest.raises(ValueError):
            to_camera(*args)


# ------------------------------------------------------------------ geometry against the rasterizer
@pytest.mark.parametrize("name", ["box", "sphere"])
@pytest.mark.parametrize("corners", [False, True])
def test_crop_is_the_view_of_the_crop_camera(name, corners):
    """A mesh rendered at its true pose (R, t) in the frame and warped by frame_crops, against the mesh rendered at
    (R_v R, R_v t) with K_v at S x S: the two silhouettes agree to IoU >= 0.97.  frame_crops cuts around the mask's t0,
    not the true t, so the object sits at R_v t in the crop camera; with t0 = t that is (0, 0, |t|).  The same render
    without R_v (at (R, R_v t)) shows what the uncorrected rotation does."""
    from nope_b200.crop import crop_intrinsics, frame_crops
    from nope_b200.vsd import render_depth
    mesh, d = make_mesh(name)
    n = 8
    R, t, masks = _scene(mesh, 5 + corners, n, corners)
    crops, t0, Rv, _ = frame_crops(_frames(masks), masks, K3, d)
    sil = (crops[:, 0] > 0).cpu()
    pose0 = torch.eye(4, dtype=torch.float64).repeat(n, 1, 1)
    pose0[:, :3, 3] = t0.cpu()
    Kv = crop_intrinsics(pose0, 1.2 * d, S).numpy()
    Rvh = Rv.cpu().numpy()
    ious, raw = [], []
    for b in range(n):
        tv = Rvh[b] @ t[b]
        for Rb, out in ((Rvh[b] @ R[b], ious), (R[b], raw)):
            r = render_depth(mesh, torch.from_numpy(pose(Rb, tv)), Kv[b], (S, S))[0].cpu() > 0
            out.append(float((r & sil[b]).sum()) / float((r | sil[b]).sum()))
    tilt = [math.degrees(math.acos(min(1.0, (np.trace(Rvh[b]) - 1) / 2))) for b in range(n)]
    print(f"{name} corners={corners}: IoU min {min(ious):.4f}, without R_v min {min(raw):.4f}, "
          f"R_v angles {min(tilt):.1f} ... {max(tilt):.1f} deg")
    assert min(ious) >= 0.97, ious
    if corners:
        assert min(tilt) > 15.0
        if name == "box":                                    # a sphere's silhouette does not show its rotation
            assert np.mean(raw) < np.mean(ious)


# ------------------------------------------------------------------ predict_pose_frames
def _detections(n=3, seed=7):
    """three detections of two objects (ids 91: box, 92: sphere) in two frames; detections 0 and 1 share frame 0
    -> (meshes {id: (mesh, d)}, ids, R [n, 3, 3], t [n, 3], masks, frames [2, H, W, 3], frame_idx)"""
    from nope_b200.vsd import render_depth
    meshes = {91: make_mesh("box"), 92: make_mesh("sphere")}
    ids = [91, 92, 91]
    rng = np.random.default_rng(seed)
    spots = [(150.0, 130.0, 700.0), (560.0, 380.0, 900.0), (400.0, 250.0, 600.0)]
    R = np.stack([rot(rng) for _ in ids])
    t = np.stack([np.linalg.solve(K3, [u, v, 1.0]) * z for u, v, z in spots])
    masks = torch.stack([(render_depth(meshes[i][0], torch.from_numpy(pose(R[b], t[b])), K3, (H, W))[0] > 0)
                         .to(torch.uint8) * 255 for b, i in enumerate(ids)])
    frames = torch.stack([_frames(masks[0] | masks[1]), _frames(masks[2])])
    return meshes, ids, R, t, masks, frames, torch.tensor([0, 0, 1])


def test_frames_to_pose_with_the_true_crop_rotation():
    """the search stubbed to return the true crop-camera rotation R_v R: predict_pose_frames returns R to 1e-12, its t
    is estimate_translation's from t0 for that R, and the MSSD that eval_bop computes (bop.pose_errors) equals the
    true rotation's at that t"""
    from nope_b200 import bop, translation
    from nope_b200.crop import frame_crops, to_crop
    from nope_b200.model import PoseConditional
    meshes, ids, R, t, masks, frames, fi = _detections()
    model = with_objects(PoseConditional(types.SimpleNamespace(device=torch.device("cuda", 0))), meshes)
    d = np.array([meshes[i][1] for i in ids])
    _, t0, Rv, _ = frame_crops(frames, masks, K3, d, frame_idx=fi)
    k = 2
    R_crop = to_crop(torch.from_numpy(R).cuda()[:, None].expand(3, k, 3, 3), Rv)

    def search(query, reference, all_relativeR, template_poses, k, angles):
        assert query.shape == (3, 3, S, S) and (angles, k) == (36, 2)
        zeros = torch.zeros((3, k), dtype=torch.int64, device="cuda")
        return R_crop, zeros, zeros, torch.zeros((3, angles, 4), device="cuda")
    model.predict_pose_inplane = search
    out = model.predict_pose_frames(frames, masks, K3, ids, torch.zeros(1, 3, S, S), torch.zeros(1, 4, 6),
                                    torch.zeros(4, 3, 3), k=k, frame_idx=fi)
    assert out["R"].shape == (3, k, 3, 3) and out["t"].shape == (3, k, 3) and out["iou"].shape == (3, k)
    assert (out["R"].cpu() - torch.from_numpy(R)[:, None]).abs().max() <= 1e-12
    assert torch.equal(out["t0"], t0) and torch.equal(out["R_crop"], R_crop)
    for b, i in enumerate(ids):
        tb, ib = translation.estimate_translation(meshes[i][0], out["R"][b:b + 1], K3, masks[b:b + 1],
                                                  t_init=t0[b:b + 1])
        assert torch.equal(out["t"][b], tb[0]) and torch.equal(out["iou"][b], ib[0])
        e_est, _ = bop.pose_errors(meshes[i][0].vertices, out["R"][b:b + 1], out["t"][b:b + 1], R[b:b + 1],
                                   t[b:b + 1], K3, model.bop_models[i]["symmetries"])
        e_true, _ = bop.pose_errors(meshes[i][0].vertices, torch.from_numpy(R[b:b + 1, None]).expand(1, k, 3, 3),
                                    out["t"][b:b + 1], R[b:b + 1], t[b:b + 1], K3, model.bop_models[i]["symmetries"])
        assert (e_est - e_true).abs().max() <= 1e-9
    assert (out["iou"] > 0.9).all()
    t_err = (out["t"].cpu() - torch.from_numpy(t)[:, None]).norm(dim=2)
    print(f"true rotation: |t - t_true| max {float(t_err.max()):.2f} mm, IoU min {float(out['iou'].min()):.4f}")


@pytest.fixture(scope="module")
def engine_scene():
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from oracle import inputs
    _, r = inputs.make_images(seed=4, batch=1)
    return {"ref": r.cuda(), "rel": synthetic_pose_batch(42, 1)[0].cuda(),
            "tp": torch.from_numpy(icosphere_object_rotations(0))}


def _chain(model, meshes, ids, frames, masks, fi, sc, refine, refiner=None):
    """frame_crops -> predict_pose_inplane (or predict_pose_inplane_refined) -> to_camera -> estimate_translation
    (-> refine_pose_contour), by hand"""
    from nope_b200 import contour_refine, translation
    from nope_b200.crop import frame_crops, to_camera
    d = np.array([meshes[i][1] for i in ids])
    crops, t0, Rv, _ = frame_crops(frames, masks, K3, d, frame_idx=fi)
    if refiner is None:
        R_crop, n, a, sim = model.predict_pose_inplane(crops, sc["ref"], sc["rel"], sc["tp"], k=3, angles=6)
        score = sim.reshape(3, -1).gather(1, a * 42 + n)
    else:
        R_crop, _, _, score = model.predict_pose_inplane_refined(crops, sc["ref"], sc["rel"], refiner, k=3)
    R = to_camera(R_crop, Rv)
    t, iou = torch.empty(3, 3, 3, dtype=torch.float64, device="cuda"), torch.empty(3, 3, dtype=torch.float64,
                                                                                   device="cuda")
    R_out = R.clone()
    for i in sorted(set(ids)):
        rows = [b for b, j in enumerate(ids) if j == i]
        tt, ii = translation.estimate_translation(meshes[i][0], R[rows], K3, masks[rows], t_init=t0[rows])
        if refine:
            R_out[rows], tt, fit = contour_refine.refine_pose_contour(meshes[i][0], R[rows], tt, K3, masks[rows])
            ii = fit["iou"]
        t[rows], iou[rows] = tt, ii
    return {"R": R_out, "t": t, "score": score, "iou": iou, "R_crop": R_crop, "t0": t0, "crops": crops}


@pytest.mark.parametrize("refine,refined_search", [(None, False), ("contour", False), (None, True)])
def test_predict_pose_frames_equals_the_chain(gpu_model, engine_scene, refine, refined_search):
    from nope_b200.inplane_refine import InplaneRefiner
    meshes, ids, _, _, masks, frames, fi = _detections()
    model = with_objects(gpu_model, meshes)
    sc = engine_scene
    refiner = InplaneRefiner(sc["tp"], angles=6, steps=2) if refined_search else None
    out = model.predict_pose_frames(frames, masks, K3, ids, sc["ref"], sc["rel"], sc["tp"], angles=6, k=3,
                                    refiner=refiner, refine=refine, frame_idx=fi)
    ref = _chain(model, meshes, ids, frames, masks, fi, sc, refine, refiner)
    for key in ("R", "t", "score", "iou", "R_crop", "t0", "crops"):
        assert torch.equal(out[key], ref[key]), key
    # the shared frame against duplicated frames
    dup = model.predict_pose_frames(frames[fi.tolist()], masks, K3, ids, sc["ref"], sc["rel"], sc["tp"], angles=6, k=3,
                                    refiner=refiner, refine=refine)
    for key in out:
        assert torch.equal(out[key], dup[key]), key


def test_synchronisations(gpu_model, engine_scene):
    """predict_pose_frames synchronises as often as its stages do on their own, and frame_crops once (its copy of
    t0).  Sync debug mode sees synchronisation on the Python / torch side only."""
    from nope_b200 import translation
    from nope_b200.crop import frame_crops, to_camera
    meshes, ids, _, _, masks, frames, fi = _detections()
    model = with_objects(gpu_model, meshes)
    sc = engine_scene
    tp = sc["tp"].cuda()
    args = (frames, masks, K3, ids, sc["ref"], sc["rel"], tp)
    model.predict_pose_frames(*args, angles=6, k=3, frame_idx=fi)            # warm-up
    _, n_all = count_host_syncs(lambda: model.predict_pose_frames(*args, angles=6, k=3, frame_idx=fi))
    d = np.array([meshes[i][1] for i in ids])
    (crops, t0, Rv, _), n_crop = count_host_syncs(lambda: frame_crops(frames, masks, K3, d, frame_idx=fi))
    (R_crop, *_), n_search = count_host_syncs(lambda: model.predict_pose_inplane(crops, sc["ref"], sc["rel"], tp, k=3,
                                                                                  angles=6))
    R, n_rot = count_host_syncs(lambda: to_camera(R_crop, Rv))
    n_fit = 0
    for i in sorted(set(ids)):
        rows = torch.tensor([b for b, j in enumerate(ids) if j == i]).cuda()
        _, n = count_host_syncs(lambda: translation.estimate_translation(
            meshes[i][0], R[rows], K3[None].repeat(len(rows), 0), masks[rows], t_init=t0[rows]))
        n_fit += n
    print(f"syncs: predict_pose_frames {n_all}, frame_crops {n_crop}, search {n_search}, to_camera {n_rot}, "
          f"fits {n_fit}")
    assert n_crop == 1 and n_rot == 0
    assert n_all == n_crop + n_search + n_fit
