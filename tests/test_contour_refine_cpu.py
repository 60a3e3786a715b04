"""CPU: the contour refinement of DESIGN.md section 20.  The numpy oracle's distance transform against a brute-force
minimum (masks touching the frame border, one pixel, empty, full); the oracle end to end on small frames rendered by
oracle/render_oracle: the true pose kept bit for bit, an image-plane shift and a change of distance corrected in the
right direction, a small rotation recovered; fewer than 6 pairs keep the pose; the default schedule; the Python
argument errors and the C ABI's refusals."""
import math

import numpy as np
import pytest

import contour_refine_oracle as cro
import translation_oracle as to
from _scenes import angle, rotvec
from oracle import render_oracle as ro

K4 = np.array([150.0, 151.0, 48.2, 35.9])                    # the 96 x 72 intrinsics of tests/test_bop_gpu.py
SIZE = (72, 96)


def _brute_force(mask):
    """(d2_out, d2_in) by the definition: the minimum over every feature pixel, -1 where the frame has none"""
    m = np.asarray(mask) != 0
    H, W = m.shape
    rr, cc = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    out = []
    for feature in (m, ~m):
        fr, fc = np.nonzero(feature)
        if len(fr) == 0:
            out.append(np.full((H, W), -1))
            continue
        d2 = (rr[..., None] - fr) ** 2 + (cc[..., None] - fc) ** 2
        out.append(d2.min(-1))
    return out


def _masks():
    rng = np.random.default_rng(0)
    yield (rng.random((9, 11)) < 0.3)
    yield (rng.random((13, 7)) < 0.85)
    m = np.zeros((10, 12), bool)
    m[0:4, 0:3] = True                                        # touches two borders
    m[7:, 9:] = True                                          # and the opposite corner
    yield m
    m = np.zeros((8, 9), bool)
    m[3, 5] = True                                            # one pixel
    yield m
    m = np.zeros((6, 40), bool)
    m[:, 17:19] = True                                        # a band from border to border
    yield m
    yield np.zeros((5, 6), bool)                              # empty
    yield np.ones((5, 6), bool)                               # full
    yield ro.render(*ro.box(), to.pose(ro.look_pose(0.3, 0.2, 0.1)[:3, :3], [3.0, -2.0, 330.0]), K4, SIZE)[0]\
        .numpy() > 0


# ------------------------------------------------------------------ the signed distance field
def test_squared_distances_equal_brute_force():
    for m in _masks():
        a_out, a_in = cro.sq_distances(m)
        b_out, b_in = _brute_force(m)
        assert np.array_equal(a_out, b_out) and np.array_equal(a_in, b_in), m.astype(int)
        assert (a_out[m] == 0).all() and (a_in[~m] == 0).all()


def test_sdf_values():
    for m in _masks():
        phi = cro.sdf(m)
        if not m.any() or m.all():
            assert np.isnan(phi).all()
            continue
        d_out, d_in = _brute_force(m)
        assert np.array_equal(phi[~m], np.sqrt(d_out[~m].astype(np.float64)) - 0.5)
        assert np.array_equal(phi[m], 0.5 - np.sqrt(d_in[m].astype(np.float64)))
        assert (phi[m] <= -0.5).all() and (phi[~m] >= 0.5).all()


def test_contour_pixels():
    D = np.zeros((6, 7), np.float32)
    D[1:5, 1:6] = 300.0                                       # a 4 x 5 block
    D[0, 3] = 300.0                                           # on the border: never a contour pixel, and it makes
    expect = D > 0                                            # (1, 3) an interior pixel of the render
    expect[0, 3] = expect[1, 3] = False
    expect[2:4, 2:5] = False
    assert np.array_equal(cro.contour(D), expect) and expect.sum() == 13


# ------------------------------------------------------------------ the oracle end to end
def _setup(R_true, t_true, mesh=None):
    v, f = ro.box() if mesh is None else mesh
    render = to.cpu_renderer(v, f, K4, SIZE)
    mask = render(R_true, t_true) > 0
    return render, mask, float(np.sqrt((np.asarray(v, np.float32).astype(np.float64) ** 2).sum(1)).max())


R_BOX = ro.look_pose(0.5, -0.4, 0.3)[:3, :3].astype(np.float64)
T_BOX = np.array([4.0, -3.0, 330.0])


def test_oracle_keeps_the_true_pose_bit_for_bit():
    render, mask, rho = _setup(R_BOX, T_BOX)
    R, t, fit, sums = cro.refine(render, R_BOX, T_BOX, mask, K4, [0.15, 0.08, 0.04, 0.02], rho)
    assert np.array_equal(R, R_BOX) and np.array_equal(t, T_BOX)
    assert (sums[21:28] == 0).all() and fit[0] == sums[-1] == fit[1] > 20
    assert fit[2] == 0.0 and fit[3] == 1.0


@pytest.mark.parametrize("axis", [0, 1])
def test_an_image_plane_shift_moves_x_and_y_back(axis):
    render, mask, rho = _setup(R_BOX, T_BOX)
    for sign in (1.0, -1.0):
        t0 = T_BOX.copy()
        t0[axis] += sign * 4.0
        R1, t1, _, _ = cro.refine(render, R_BOX, t0, mask, K4, [0.3, 0.3], rho)
        assert sign * (t1[axis] - t0[axis]) < -1.0, (t0, t1)
        R, t, fit, _ = cro.refine(render, R_BOX, t0, mask, K4, cro_default(), rho)
        assert np.abs(t - T_BOX).max() < 1.0 and abs(t[axis] - T_BOX[axis]) < 0.5, t - T_BOX
        assert fit[3] > 0.95


def test_a_scale_about_the_origin_moves_z():
    render, mask, rho = _setup(R_BOX, T_BOX)
    for s in (1.06, 0.95):
        t0 = T_BOX * s
        _, t1, _, _ = cro.refine(render, R_BOX, t0, mask, K4, [0.3, 0.3], rho)
        assert abs(t1[2] - T_BOX[2]) < abs(t0[2] - T_BOX[2]) - 3.0, (t0, t1)
        _, t, _, _ = cro.refine(render, R_BOX, t0, mask, K4, cro_default(), rho)
        assert abs(t[2] - T_BOX[2]) < 0.25 * abs(t0[2] - T_BOX[2]), t - T_BOX


def test_oracle_recovers_a_small_rotation():
    render, mask, rho = _setup(R_BOX, T_BOX)
    R0 = rotvec([0.03, -0.02, 0.025]) @ R_BOX
    R, t, fit, _ = cro.refine(render, R0, T_BOX, mask, K4, cro_default(), rho)
    assert angle(R, R_BOX) < 0.5 * angle(R0, R_BOX), (angle(R0, R_BOX), angle(R, R_BOX))
    assert fit[3] > 0.95


def cro_default():
    from nope_b200.contour_refine import default_tau
    return default_tau()


def test_fewer_than_six_pairs_or_a_camera_behind_keep_the_pose():
    R, t = np.eye(3), np.array([1.0, 2.0, 300.0])
    sums = np.zeros(29, dtype=np.int64)
    sums[-1] = 5
    for q in range(6):
        sums[cro.dro.UPPER.index((q, q))] = 1 << 32
    sums[21] = 1 << 30
    R1, t1 = cro.solve(sums, R, t, 2.0, K4, 50.0)
    assert np.array_equal(R1, R) and np.array_equal(t1, t)
    sums[-1] = 6
    R1, t1 = cro.solve(sums, R, t, 2.0, K4, 50.0)
    assert not np.array_equal(R1, R)
    R2, t2 = cro.solve(sums, R, t * [1, 1, -1], 2.0, K4, 50.0)
    assert np.array_equal(R2, R) and np.array_equal(t2, t * [1, 1, -1])


def test_masks_without_a_contour_keep_the_pose():
    render, _, rho = _setup(R_BOX, T_BOX)
    t0 = T_BOX + [2.0, 1.0, 5.0]
    for mask in (np.zeros(SIZE, bool), np.ones(SIZE, bool)):
        R, t, fit, sums = cro.refine(render, R_BOX, t0, mask, K4, [0.1, 0.1, 0.1], rho)
        assert np.array_equal(R, R_BOX) and np.array_equal(t, t0) and (sums == 0).all()
        assert fit[0] == 0 and fit[1] > 0 and np.isnan(fit[2]) and np.isnan(fit[3])


# ------------------------------------------------------------------ the default schedule
def test_default_tau_schedule():
    from nope_b200.contour_refine import DEFAULT_ITERS, TAU_END, TAU_START, default_tau
    assert default_tau().shape == (DEFAULT_ITERS + 1,)
    for iters in (0, 1, DEFAULT_ITERS, 10):
        tau = default_tau(iters)
        assert tau.shape == (iters + 1,) and np.isclose(tau[-1], TAU_END)
        if iters:
            assert np.isclose(tau[0], TAU_START) and (np.diff(tau) < 0).all()
            assert np.allclose(tau[1:] / tau[:-1], (TAU_END / TAU_START) ** (1 / iters))
    for bad in (-1, 1.5, 2000, True):
        with pytest.raises(ValueError):
            default_tau(bad)
    assert np.allclose(default_tau(4, 0.3, 0.05)[[0, -1]], [0.3, 0.05])
    for bad in ((0.0, 0.02), (0.15, -1.0), (np.inf, 0.02), (0.15, np.nan)):
        with pytest.raises(ValueError):
            default_tau(4, *bad)


# ------------------------------------------------------------------ argument errors
def test_argument_errors():
    from nope_b200 import _lib
    from nope_b200.contour_refine import mask_sdf, refine_pose_contour
    from nope_b200.vsd import Mesh
    v, f = ro.box()
    mesh = Mesh(v, f, device="cpu")
    F = 2
    R, t = np.eye(3)[None].repeat(F, 0), np.tile([0.0, 0.0, 300.0], (F, 1))
    M = np.zeros((F, 8, 10), np.uint8)
    ok = dict(mesh=mesh, R=R, t=t, K=K4, masks=M)
    with pytest.raises(_lib.NopeError):                          # no CPU fallback
        refine_pose_contour(**ok)
    for bad in (dict(mesh=(v, f)), dict(R=R[:, :2]), dict(R=R.astype(np.int32)), dict(t=t[:, :2]), dict(t=t[:1]),
                dict(masks=M[:1]), dict(masks=M.astype(np.float32)), dict(masks=M[0, 0]),
                dict(masks=np.zeros((F, 8, 9000), np.uint8)), dict(iters=-1), dict(iters=1.5), dict(iters=2000),
                dict(tau=[0.1, 0.2]), dict(tau=0.0), dict(tau=np.inf), dict(tau=-0.1), dict(znear=0.0),
                dict(K=np.ones((3, 4))), dict(K=K4 * [0, 1, 1, 1])):
        with pytest.raises(ValueError):
            refine_pose_contour(**{**ok, **bad})
    with pytest.raises(ValueError):
        refine_pose_contour(**ok, iters=2, tau=[0.3, 0.2, -1.0])
    for bad in (M.astype(np.float32), M[0, 0], np.zeros((1, 8200, 4), np.uint8)):
        with pytest.raises(ValueError):
            mask_sdf(bad)


def test_c_abi_refuses_bad_arguments():
    """every refusal happens before any CUDA call, so it holds without a GPU"""
    from nope_b200 import _lib
    lib = _lib.load()
    K = np.array([[150.0, 151.0, 48.0, 36.0]])
    tau = np.array([0.2, 0.1, 0.05])

    def call(F=1, P=1, H=8, W=8, iters=2, znear=0.05, k=K, null=None, V=3, NF=1, rho=50.0, tv=tau):
        args = [1, V, 1, NF, 1, 1, 1, k.ctypes.data, F, P, H, W, rho, tv.ctypes.data, iters, znear, 1, 1, 1, 1, None,
                None]
        if null is not None:
            args[null] = None
        return lib.nope_refine_contour_occluded(*args[:7], None, *args[7:])     # occluders NULL
    for kw in (dict(F=0), dict(F=65536), dict(P=0), dict(P=65536), dict(H=0), dict(W=8193), dict(iters=-1),
               dict(iters=1025), dict(znear=0.0), dict(znear=math.inf), dict(rho=0.0), dict(rho=-1.0),
               dict(rho=math.nan), dict(tv=tau * [1, 1, 0]), dict(tv=tau * [1, -1, 1]), dict(tv=tau * [np.nan, 1, 1]),
               dict(k=K * [np.nan, 1, 1, 1]), dict(k=K * [1, 0, 1, 1]), dict(k=K * [1, 1, np.inf, 1]), dict(V=0),
               dict(NF=0), dict(null=0), dict(null=2), dict(null=4), dict(null=5), dict(null=6), dict(null=7),
               dict(null=13), dict(null=16), dict(null=17), dict(null=18), dict(null=19)):
        with pytest.raises(_lib.NopeError):
            _lib.check(call(**kw))

    def sdf(masks=1, F=1, H=8, W=8, out=1):
        return lib.nope_mask_sdf(masks, F, H, W, out, None)
    for kw in (dict(masks=None), dict(out=None), dict(F=0), dict(F=65536), dict(H=0), dict(H=8193), dict(W=0),
               dict(W=8193)):
        with pytest.raises(_lib.NopeError):
            _lib.check(sdf(**kw))
