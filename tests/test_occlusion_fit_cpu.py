"""CPU: the pose fits under occlusion of DESIGN.md section 24.  The oracle's fixed point at the true pose on small
scenes rendered by oracle/render_oracle, with a nearer occluder and an object behind the target; occluders built from
a frame's detections; and argument refusals in Python and through the C ABI."""
import numpy as np
import pytest
import torch

import contour_refine_oracle as cro
import occlusion_fit_oracle as ofo
import translation_oracle as to
from oracle import render_oracle as ro

K4 = np.array([150.0, 151.0, 48.2, 35.9])                    # 96 x 72
SIZE = (72, 96)
TAUS = np.geomspace(0.15, 0.02, 4)


def _scene(shift):
    """a box target at 360 mm, a sphere occluder 120 mm nearer moved `shift` px to the right of the target's centre,
    and a box 150 mm behind the target -> (render, R, t, M visible, O occluder, O_behind)"""
    v, f = ro.box()
    render = to.cpu_renderer(v, f, K4, SIZE)
    R = ro.look_pose(0.4, -0.3, 0.2)[:3, :3].astype(np.float64)
    t = np.array([4.0, -3.0, 360.0])
    D = render(R, t)
    zo = 240.0
    to_ = np.array([t[0] / t[2] * zo + shift * zo / K4[0], t[1] / t[2] * zo, zo])
    vs, fs = ro.sphere(14.0, 1)
    Do = to.cpu_renderer(vs, fs, K4, SIZE)(np.eye(3), to_)
    Db = to.cpu_renderer(*ro.box(60.0, 40.0, 10.0), K4, SIZE)(np.eye(3), np.array([30.0, 10.0, 510.0]))
    M = (D > 0) & ~((Do > 0) & (Do < D))
    return render, R, t, M, Do > 0, Db > 0


@pytest.mark.parametrize("shift", [-11.0, 10.0])
def test_the_true_pose_is_a_fixed_point_under_occlusion(shift):
    """with M = the target's visible pixels and O the occluder's silhouette (alone, or with an object behind the
    target), the true pose stays put in both fits with IoU 1; without O the translation fit leaves it"""
    render, R, t, M, O, Ob = _scene(shift)
    cover = (M != (render(R, t) > 0)).sum() / (render(R, t) > 0).sum()
    assert 0.1 < cover < 0.8, cover
    assert (Ob & M).sum() > 20                                     # O also takes some of the target's visible pixels
    for occ in (O, O | Ob):
        t1, iou, _ = ofo.fit_translation(render, R, t, M, occ, K4, 3)
        assert np.abs(t1 - t).max() <= 1e-6 and iou == 1.0, (t1, t, iou)
        R2, t2, fit, sums = cro.refine(render, R, t, M, K4, TAUS, 40.0, occ=occ)
        assert np.array_equal(R2, R) and np.array_equal(t2, t) and fit[3] == 1.0, fit
        assert fit[0] >= 6 and fit[1] >= fit[0] and fit[2] == 0.0
    t1, iou, _ = to.fit(render, R, t, M, K4, 3)                  # the visible mask alone pulls the fit away
    assert np.abs(t1 - t).max() > 1.0 and iou < 1.0


def test_an_all_zero_occluder_is_the_plain_fit():
    render, R, t, M, _, _ = _scene(10.0)
    zero = np.zeros_like(M)
    t0 = t + [2.0, -1.5, 12.0]
    a, b = ofo.fit_translation(render, R, t0, M, zero, K4, 3), to.fit(render, R, t0, M, K4, 3)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2]
    a, b = cro.refine(render, R, t0, M, K4, TAUS, 40.0, occ=zero), cro.refine(render, R, t0, M, K4, TAUS, 40.0)
    assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


def test_contour_pixels_next_to_an_occluder_are_not_counted():
    D = np.zeros((9, 12), np.float32)
    D[2:7, 3:9] = 500.0
    occ = np.zeros((9, 12), np.uint8)
    occ[4, 9] = 1                                                 # right of the right edge's middle pixel
    cont = cro.contour(D)
    assert cont[4, 8] and cro.known4(occ).sum() == 9 * 12 - 5
    phi = cro.sdf(cro.visible(D > 0, occ))
    _, nc = cro.accumulate(D, phi, K4, np.array([0.0, 0.0, 500.0]), 3.0, 40.0, occ)
    assert nc == cont.sum() - 1


# ------------------------------------------------------------------ occluders from a frame's detections
def _hand_masks():
    m = np.zeros((5, 6, 7), np.uint8)
    m[0, 1:4, 1:4] = 1
    m[1, 2:5, 3:6] = 255                                           # overlaps detection 0 (same frame)
    m[2, 0:2, 0:7] = 1                                             # frame 0 too
    m[3, 1:5, 1:5] = 1                                             # alone in frame 2
    m[4, 3:6, 2:6] = 1                                             # frame 1, with nobody else
    return m


@pytest.mark.parametrize("as_bool", [False, True])
def test_detection_occluders(as_bool):
    from nope_b200.crop import detection_occluders
    m = _hand_masks()
    fi = np.array([0, 0, 0, 2, 1])
    got = detection_occluders(torch.from_numpy(m.astype(bool) if as_bool else m), torch.from_numpy(fi), num_frames=3)
    assert got.dtype == torch.uint8 and got.shape == m.shape
    want = ofo.detection_occluders(m, fi)
    assert np.array_equal(got.numpy(), want)
    assert not want[3].any() and not want[4].any()                # a detection alone in its frame
    assert want[0].any() and not (want[0] & m[0]).any()           # O never covers the detection's own mask
    assert np.array_equal(detection_occluders(m, fi).numpy(), want)          # num_frames from frame_idx
    assert not detection_occluders(m).numpy().any()                # one frame per detection
    # indices outside [0, F) fall into the groups below 0 and at F: no out-of-range write
    fi2 = np.array([-3, -1, 7, 5, 0])
    assert np.array_equal(detection_occluders(m, fi2, num_frames=3).numpy(),
                          ofo.detection_occluders(m, np.clip(fi2, -1, 3)))
    for bad in (dict(frame_idx=fi[:4]), dict(frame_idx=fi.astype(np.float32)), dict(masks=m.astype(np.float32)),
                dict(masks=m[0]), dict(frame_idx=fi, num_frames=0)):
        with pytest.raises(ValueError):
            detection_occluders(**{"masks": m, **bad})


# ------------------------------------------------------------------ refusals
def test_python_refuses_bad_occluders():
    from nope_b200 import _lib
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import occluder_masks
    from nope_b200.vsd import Mesh
    M = np.zeros((2, 8, 10), np.uint8)
    assert occluder_masks(None, torch.from_numpy(M)) is None
    assert occluder_masks(M[:1, None, 0].repeat(8, 1), torch.from_numpy(M[:1])).shape == (1, 8, 10)
    for bad in (M[:1], M[:, :, :9], M.astype(np.float32), M[0, 0]):
        with pytest.raises(ValueError):
            occluder_masks(bad, torch.from_numpy(M))
    v, f = ro.box()
    ok = dict(mesh=Mesh(v, f, device="cpu"), R=np.eye(3)[None].repeat(2, 0), t=np.tile([0.0, 0.0, 300.0], (2, 1)),
              K=K4, masks=M)
    for bad in (M[:1], M[:, :7], M.astype(np.int32)):
        with pytest.raises(ValueError):
            refine_pose_contour(**ok, occluders=bad)
    with pytest.raises(_lib.NopeError):                          # checked, then no CPU fallback
        refine_pose_contour(**ok, occluders=M.astype(bool))


def test_c_abi_refuses_bad_arguments():
    """the occluded entry points refuse what the plain ones refuse, before any CUDA call, with or without occluders"""
    from nope_b200 import _lib
    lib = _lib.load()
    K = np.array([[150.0, 151.0, 48.0, 36.0]])
    tau = np.array([0.2, 0.1, 0.05])

    def fit(occ, F=1, H=8, znear=0.05, k=K, null=None):
        args = [1, 3, 1, 1, 1, 1, 1, occ, k.ctypes.data, F, 1, H, 8, znear, 2, 1, 1, 1, None, None]
        if null is not None:
            args[null] = None
        return lib.nope_fit_translation_occluded(*args)

    def contour(occ, F=1, H=8, znear=0.05, k=K, null=None, rho=50.0, tv=tau):
        args = [1, 3, 1, 1, 1, 1, 1, occ, k.ctypes.data, F, 1, H, 8, rho, tv.ctypes.data, 2, znear, 1, 1, 1, 1, None,
                None]
        if null is not None:
            args[null] = None
        return lib.nope_refine_contour_occluded(*args)
    for occ in (None, 1):
        for kw in (dict(F=0), dict(F=65536), dict(H=0), dict(znear=0.0), dict(k=K * [np.nan, 1, 1, 1]), dict(null=0),
                   dict(null=2), dict(null=4), dict(null=5), dict(null=6), dict(null=8)):
            with pytest.raises(_lib.NopeError):
                _lib.check(fit(occ, **kw))
            with pytest.raises(_lib.NopeError):
                _lib.check(contour(occ, **kw))
        for kw in (dict(null=15), dict(null=16), dict(null=17)):
            with pytest.raises(_lib.NopeError):
                _lib.check(fit(occ, **kw))
        for kw in (dict(rho=0.0), dict(tv=tau * [1, 0, 1]), dict(null=14), dict(null=17), dict(null=18),
                   dict(null=19), dict(null=20)):
            with pytest.raises(_lib.NopeError):
                _lib.check(contour(occ, **kw))
    if torch.cuda.is_available():
        return                                                    # the accepted call below would run on fake pointers
    refusals = ("null argument", "must be", "iters")
    for call in (fit, contour):
        assert call(None) != 0                                    # accepted, then no device to run on
        msg = lib.nope_last_error().decode()
        assert msg and not any(r in msg for r in refusals), msg


def test_abi_version_and_symbols_bind():
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_abi_version() == 3
    for name in ("nope_fit_translation_occluded", "nope_refine_contour_occluded"):
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
