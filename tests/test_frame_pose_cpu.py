"""CPU: the crop camera (DESIGN.md section 23) without a device.  The oracle's R_v is a rotation that looks along the
ray to the object; K_v R_v maps crop_frame's square onto the crop's corners; the homography K_v R_v K^-1 agrees with
crop_transforms' forward map up to the int32 truncation of the corners; bad arguments are refused through the C ABI and in Python before any device work."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import crop_camera_oracle as cco

K = np.array([[1075.65091572, 0.0, 360.0], [0.0, 1073.90347929, 270.0], [0.0, 0.0, 1.0]])   # Primesense 720 x 540
S = 256


def _poses(keep_inplane, F=400, seed=None):
    """seeded poses in mm; the keep_inplane=False rule expects metres (crop_transforms), so its translations are
    scaled to metres"""
    P = cco.seeded_poses(1 if seed is None else seed, F, keep_inplane, K)
    if not keep_inplane:
        P[:, :3, 3] /= 1000.0
    return P


def _square(pose, keep_inplane, s):
    """crop_frame's w1 ... w4 (before projection), as nope_b200.crop._corners builds them"""
    o, upper, right = cco._vectors(pose, keep_inplane)
    o, upper, right = np.array(o), np.array(upper), np.array(right)
    upper = upper * (s / 2) / np.linalg.norm(upper)
    right = right * (s / 2) / np.linalg.norm(right)
    return [o + upper - right, o - upper - right, o + upper + right, o - upper + right]


@pytest.mark.parametrize("keep_inplane", [True, False])
def test_oracle_is_a_rotation_along_the_ray(keep_inplane):
    P = _poses(keep_inplane)
    Rv = cco.crop_camera(P, keep_inplane)
    eye = np.eye(3)
    assert np.abs(Rv @ Rv.transpose(0, 2, 1) - eye).max() <= 1e-15
    assert np.abs(np.linalg.det(Rv) - 1).max() <= 1e-15
    o = P[:, :3, 3]
    ro = np.einsum("fij,fj->fi", Rv, o)
    n = np.linalg.norm(o, axis=1)
    assert np.abs(ro[:, :2]).max() <= 1e-15 * n.max() * 4 and np.abs(ro[:, 2] / n - 1).max() <= 1e-15


def test_on_axis_and_fallback_give_identity():
    p = np.eye(4)
    p[2, 3] = 700.0
    assert np.array_equal(cco.crop_camera(p, True), np.eye(3))
    # keep_inplane=False on the axis with R = I: the world's up lies along o, crop_frame falls back to image axes
    p[2, 3] = 0.7
    o, upper, right = cco._vectors(p, False)
    assert np.linalg.norm(upper) == 0 and np.linalg.norm(right) == 0
    assert np.array_equal(cco.crop_camera(p, False), np.eye(3))


@pytest.mark.parametrize("keep_inplane", [True, False])
def test_ideal_camera_maps_the_square_onto_the_crop(keep_inplane):
    P = _poses(keep_inplane, 200)
    s = 0.12 if not keep_inplane else 120.0
    Rv = cco.crop_camera(P, keep_inplane)
    target = np.array([[0, 0], [0, S], [S, 0], [S, S]], dtype=np.float64)
    worst = 0.0
    for f in range(len(P)):
        Kv = cco.intrinsics(P[f], s, S)
        for w, q in zip(_square(P[f], keep_inplane, s), target):
            x = Kv @ Rv[f] @ w
            worst = max(worst, np.abs(x[:2] / x[2] - q).max())
    assert worst <= 1e-9, worst


@pytest.mark.parametrize("keep_inplane", [True, False])
def test_homography_agrees_with_crop_transforms(keep_inplane):
    """K_v R_v K^-1 against the cv2 map of the truncated corners, s = 1.2 x 100 mm, objects 400 ... 1200 mm deep (the
    smallest squares span about 107 px of the frame).  The crop's corners land within sqrt(2) px of each other in the
    frame (measured 1.396 and 1.387 px); over a grid of the whole crop the two maps part by at most 1.5 px in the
    frame (measured 1.37 and 1.47 px), 3.4 px in the crop.  A rotation recovered from the cv2 map alone is not that
    close: a 107 px square pins the tilt out of the image plane poorly (DESIGN.md section 23)."""
    pytest.importorskip("cv2")
    from nope_b200.crop import forward_map
    P = _poses(keep_inplane, 300, seed=5)
    s = 0.12 if not keep_inplane else 120.0
    Rv = cco.crop_camera(P, keep_inplane)
    Kinv = np.linalg.inv(K)
    corners = np.array([[0, 0, 1], [0, S, 1], [S, 0, 1], [S, S, 1]], dtype=np.float64).T
    g = np.stack(np.meshgrid(np.arange(0, S + 1, 8.0), np.arange(0, S + 1, 8.0)), -1).reshape(-1, 2)
    grid = np.concatenate([g, np.ones((len(g), 1))], 1).T
    worst_corner, worst_frame, worst_crop = 0.0, 0.0, 0.0
    for f in range(len(P)):
        Kv = cco.intrinsics(P[f], s, S)
        Hm = Kv @ Rv[f] @ Kinv
        M = forward_map(K, P[f], s, S, keep_inplane)
        a, b = np.linalg.solve(Hm, corners), np.linalg.solve(M, corners)
        worst_corner = max(worst_corner, np.linalg.norm(a[:2] / a[2] - b[:2] / b[2], axis=0).max())
        y = Hm @ np.linalg.solve(M, grid)
        d = np.linalg.norm(y[:2] / y[2] - grid[:2], axis=0).max()               # crop px
        side = K[0, 0] * s / np.linalg.norm(P[f, :3, 3])                          # the square's side in frame px
        worst_crop, worst_frame = max(worst_crop, d), max(worst_frame, d * side / S)
    print(f"keep_inplane={keep_inplane}: corners {worst_corner:.3f} px, crop grid {worst_frame:.3f} px in the frame, "
          f"{worst_crop:.3f} px in the crop")
    assert worst_corner <= math.sqrt(2) and worst_frame <= 1.5, (worst_corner, worst_frame)


def test_uncorrected_rotation_at_the_frame_corner():
    """at the corner of the 720 x 540 Primesense frame the crop camera's axis z_v is 22.7 degrees off the optical axis,
    and R_v, the error of a crop rotation taken for a camera rotation, is a 22.8 degree rotation"""
    p = np.eye(4)
    p[:3, 3] = np.linalg.solve(K, [0.0, 0.0, 1.0]) * 800.0
    Rv = cco.crop_camera(p, True)
    assert abs(math.degrees(math.acos(Rv[2, 2])) - 22.71) < 0.01
    assert abs(math.degrees(math.acos((np.trace(Rv) - 1) / 2)) - 22.82) < 0.01


def test_intrinsics_equal_the_oracle():
    from nope_b200.crop import crop_intrinsics
    P = _poses(True, 20)
    s = np.linspace(80.0, 200.0, 20)
    Kv = crop_intrinsics(torch.from_numpy(P), torch.from_numpy(s), S).numpy()
    assert Kv.shape == (20, 3, 3) and Kv.dtype == np.float64
    for f in range(20):
        assert np.array_equal(Kv[f], cco.intrinsics(P[f], s[f], S))
    assert crop_intrinsics(torch.from_numpy(P[0]), 120.0).shape == (3, 3)
    for bad in (dict(pose=torch.zeros(2, 3, 4)), dict(virtual_bbox_size=torch.ones(3)), dict(image_size=0),
                dict(image_size=1.5)):
        args = {"pose": torch.from_numpy(P[:2]), "virtual_bbox_size": 120.0, "image_size": S, **bad}
        with pytest.raises(ValueError):
            crop_intrinsics(**args)


# ------------------------------------------------------------------ ABI
def _pose_buf(F=2, **set_):
    p = np.tile(np.eye(4), (F, 1, 1))
    p[:, 2, 3] = 500.0
    for (f, i, j), v in set_.get("at", {}).items():
        p[f, i, j] = v
    return p


@pytest.mark.parametrize("keep,at,F,needle", [
    (1, {}, 0, "F must"), (1, {}, 65536, "F must"), (2, {}, 2, "keep_inplane"), (-1, {}, 2, "keep_inplane"),
    (1, {(1, 0, 3): math.nan}, 2, "finite"), (1, {(0, 2, 3): math.inf}, 2, "finite"),
    (0, {(1, 1, 1): math.nan}, 2, "finite"), (0, {(0, 2, 0): -math.inf}, 2, "finite"),
    (1, {(1, 2, 3): 0.0}, 2, "Z > 0"), (1, {(0, 2, 3): -3.0}, 2, "Z > 0")])
def test_crop_camera_refusals(keep, at, F, needle):
    """refused on the host before any CUDA call: these run without a GPU"""
    from nope_b200 import _lib
    lib = _lib.load()
    p = _pose_buf(max(F, 2), at=at)
    assert lib.nope_crop_camera(C.c_void_p(p.ctypes.data), F, keep, C.c_void_p(256), None) != 0
    assert needle in lib.nope_last_error().decode()


def test_crop_camera_null_and_rotate_refusals():
    from nope_b200 import _lib
    lib = _lib.load()
    p = _pose_buf()
    P = C.c_void_p(256)
    assert lib.nope_crop_camera(None, 2, 1, P, None) != 0 and "null" in lib.nope_last_error().decode()
    assert lib.nope_crop_camera(C.c_void_p(p.ctypes.data), 2, 1, None, None) != 0
    assert "null" in lib.nope_last_error().decode()
    args = dict(Rv=P, F=2, R=P, P=3, to=1, out=P)
    for bad, needle in ((dict(Rv=None), "null"), (dict(R=None), "null"), (dict(out=None), "null"),
                        (dict(F=0), "F and P"), (dict(F=65536), "F and P"), (dict(P=0), "F and P"),
                        (dict(P=65536), "F and P"), (dict(to=2), "to_camera"), (dict(to=-1), "to_camera")):
        a = {**args, **bad}
        assert lib.nope_crop_rotate(a["Rv"], a["F"], a["R"], a["P"], a["to"], a["out"], None) != 0
        assert needle in lib.nope_last_error().decode()


# ------------------------------------------------------------------ Python
def test_python_refusals_without_a_device():
    from nope_b200._lib import NopeError
    from nope_b200.crop import crop_camera, frame_crops, to_camera, to_crop
    pose = torch.from_numpy(_pose_buf())
    with pytest.raises(NopeError):
        crop_camera(pose)
    R = torch.eye(3, dtype=torch.float64).repeat(2, 1, 1)
    with pytest.raises(NopeError):
        to_camera(R, R)
    with pytest.raises(NopeError):
        to_crop(R, R)
    fr = torch.zeros(2, 54, 72, 3, dtype=torch.uint8)
    m = torch.zeros(2, 54, 72, dtype=torch.uint8)
    m[:, 20:30, 30:40] = 255
    good = {"frames": fr, "masks": m, "K": torch.from_numpy(K), "diameter": 100.0}
    empty = m.clone()
    empty[1] = 0
    for bad in (dict(masks=m.float()), dict(masks=m[0]), dict(K=torch.eye(2)), dict(K=torch.eye(3).repeat(3, 1, 1)),
                dict(diameter=0.0), dict(diameter=[1.0, 2.0, 3.0]), dict(diameter=math.nan), dict(masks=empty)):
        with pytest.raises(ValueError):
            frame_crops(**{**good, **bad})


def test_predict_pose_frames_refusals():
    from nope_b200.model import PoseConditional
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    m = torch.zeros(2, 54, 72, dtype=torch.uint8)
    ref = torch.zeros(1, 3, 256, 256)
    rel = torch.zeros(1, 4, 6)
    args = dict(frames=torch.zeros(2, 54, 72, 3, dtype=torch.uint8), masks=m, K=torch.from_numpy(K), obj_ids=[1, 1],
                reference=ref, all_relativeR=rel, template_poses=torch.zeros(4, 3, 3))
    with pytest.raises(ValueError, match="refine"):
        model.predict_pose_frames(**args, refine="depth")
    with pytest.raises(ValueError, match="models_info"):
        model.predict_pose_frames(**args)
    model.tless_cad[1] = object()
    model.bop_models[1] = {"diameter": 100.0}
    with pytest.raises(ValueError, match="obj_ids"):
        model.predict_pose_frames(**{**args, "obj_ids": [1]})
    with pytest.raises(ValueError, match="reference"):
        model.predict_pose_frames(**{**args, "reference": torch.zeros(3, 3, 256, 256)})
