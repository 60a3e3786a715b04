"""CPU: the depth refinement of DESIGN.md section 19.  The numpy oracle runs the full ICP on small frames rendered by
oracle/render_oracle: it recovers a known small motion of the box, keeps the true pose, does not slide a plane seen
face-on in its plane, and does not turn a sphere while its translation converges.  Also the fixed-point conversion
and its overflow bound, the default tolerance schedule, the Python argument errors, and the C ABI's refusals."""
import math

import numpy as np
import pytest
import torch

import depth_refine_oracle as dro
import translation_oracle as to
from _scenes import angle, rotvec
from oracle import render_oracle as ro

K4 = np.array([150.0, 151.0, 48.2, 35.9])                    # the 96 x 72 intrinsics of tests/test_bop_gpu.py
SIZE = (72, 96)


def _setup(v, f, R_true, t_true):
    render = to.cpu_renderer(v, f, K4, SIZE)
    S = render(R_true, t_true).astype(np.float64)
    return render, S, dro.radius(v)


# ------------------------------------------------------------------ the oracle end to end
def test_oracle_recovers_a_small_motion_of_the_box():
    v, f = ro.box()
    R_true = ro.look_pose(0.5, -0.4, 0.3)[:3, :3].astype(np.float64)
    t_true = np.array([4.0, -3.0, 330.0])
    render, S, rho = _setup(v, f, R_true, t_true)
    R0 = rotvec([0.03, -0.02, 0.025]) @ R_true
    t0 = t_true + [3.0, -2.0, 6.0]
    taus = np.geomspace(25.0, 2.0, 9)
    R, t, fit, sums = dro.refine(render, R0, t0, S, S > 0, K4, taus, rho)
    assert angle(R, R_true) < 0.1 and np.abs(t - t_true).max() < 0.1, (angle(R, R_true), t - t_true)
    assert angle(R0, R_true) > 2.0
    assert fit[0] == sums[-1] > 100 and fit[1] == np.count_nonzero(S) and 0.5 < fit[3] <= 1.0 and fit[2] < 0.05


def test_oracle_keeps_the_true_pose():
    """the sensor depth is the render at the true pose, so every residual is 0 and every update the identity"""
    v, f = ro.sphere(40.0, 1)
    R_true = ro.look_pose(0.2, 1.1, -0.7)[:3, :3].astype(np.float64)
    t_true = np.array([-6.0, 5.0, 360.0])
    render, S, rho = _setup(v, f, R_true, t_true)
    R, t, fit, sums = dro.refine(render, R_true, t_true, S, None, K4, [8.0, 4.0, 2.0], rho)
    assert np.array_equal(R, R_true) and np.array_equal(t, t_true)
    assert fit[2] == 0.0 and sums[27] == 0 and (sums[21:27] == 0).all() and fit[0] > 0


def test_oracle_does_not_slide_a_face_on_plane():
    """a plane facing the camera: its in-plane translation and its rotation about the normal are unobservable: the
    damping keeps the first update from moving them at all, later ones (after a tiny tilt) by < 1e-4 mm, while the
    distance converges"""
    v, f = ro.plane(8, 6, 120.0, 90.0)
    R_true = np.eye(3)
    t_true = np.array([0.0, 0.0, 400.0])
    render, S, rho = _setup(v, f, R_true, t_true)
    t0 = np.array([3.0, -2.0, 406.0])
    R, t, fit, sums = dro.refine(render, R_true, t0, S, None, K4, np.geomspace(20.0, 2.0, 6), rho)
    assert np.abs(t[:2] - t0[:2]).max() < 1e-4, t - t0
    assert abs(t[2] - 400.0) < 1e-3
    assert angle(R, R_true) < 1e-3
    # the first update, from an exactly face-on render: the unobservable parameters do not move at all
    R1, t1, _, _ = dro.refine(render, R_true, t0, S, None, K4, [20.0, 20.0], rho)
    assert t1[0] == t0[0] and t1[1] == t0[1] and t1[2] != t0[2]
    assert R1[0, 1] == R1[1, 0]                                  # no turn about the normal: R1[0, 1] - R1[1, 0] = -4 w z


def test_oracle_does_not_turn_a_sphere():
    """a sphere about its centre: the rotation is (almost) unobservable and does not drift while t converges"""
    v, f = ro.sphere(40.0, 1)
    R_true = ro.look_pose(0.4, -0.9, 0.2)[:3, :3].astype(np.float64)
    t_true = np.array([5.0, 2.0, 340.0])
    render, S, rho = _setup(v, f, R_true, t_true)
    t0 = t_true + [4.0, -3.0, 8.0]
    R, t, fit, _ = dro.refine(render, R_true, t0, S, None, K4, np.geomspace(20.0, 2.0, 8), rho)
    assert np.abs(t - t_true).max() < 0.3, t - t_true
    assert angle(R, R_true) < 1.0


def test_fewer_than_six_pairs_keep_the_pose():
    R, t = np.eye(3), np.array([1.0, 2.0, 3.0])
    sums = np.zeros(29, dtype=np.int64)
    sums[-1] = 5
    sums[0] = 1 << 32
    R1, t1 = dro.solve(sums, R, t, 1.0, 1.0)
    assert np.array_equal(R1, R) and np.array_equal(t1, t)


def test_empty_frame_gives_nan_fit():
    fit = dro.fit_stats(np.zeros(29, dtype=np.int64), 0, 2.0)
    assert fit[0] == 0 and fit[1] == 0 and np.isnan(fit[2]) and np.isnan(fit[3])
    fit = dro.fit_stats(np.zeros(29, dtype=np.int64), 10, 2.0)
    assert np.isnan(fit[2]) and fit[3] == 0.0


# ------------------------------------------------------------------ fixed point
def test_fixed_point_conversion_at_the_extremes():
    u = 2.0 ** -32
    assert list(dro.fixed([0.5 * u, 1.5 * u, 2.5 * u, -0.5 * u, -1.5 * u])) == [0, 2, 2, 0, -2]   # half to even
    top = 1 << 36
    assert list(dro.fixed([16.0, 1e300, np.inf, -16.0, -np.inf, 15.999999])) == \
        [top, top, top, -top, -top, int(np.rint(15.999999 * 2 ** 32))]
    assert dro.unfix(top) == 16.0 and dro.unfix(-3) == -3 * u


def test_fixed_point_sums_cannot_overflow():
    """the rasterizer's largest image has 2^26 pixels and every product is at most 2^36 units: the sum of 2^26 such
    products is <= 2^62, inside int64, whatever the order"""
    from nope_b200.vsd import MAX_SIDE
    n = MAX_SIDE * MAX_SIDE
    assert n == 2 ** 26
    big = int(dro.fixed(dro.CLAMP))
    assert big == dro.CLAMP * dro.SCALE == 2 ** 36
    assert n * big <= 2 ** 62 < 2 ** 63 - 1
    a = np.full(1 << 16, big, dtype=np.int64)
    assert int(a.sum()) * (n >> 16) == n * big                    # no wrap in int64 arithmetic either


# ------------------------------------------------------------------ the default schedule
def test_default_tau_schedule():
    from nope_b200.depth_refine import DEFAULT_ITERS, TAU_END, TAU_START, default_tau
    for iters in (0, 1, DEFAULT_ITERS, 10):
        tau = default_tau(80.0, iters)
        assert tau.shape == (iters + 1,) and np.isclose(tau[-1], TAU_END * 80.0)
        if iters:
            assert np.isclose(tau[0], TAU_START * 80.0) and (np.diff(tau) < 0).all()
            assert np.allclose(tau[1:] / tau[:-1], (TAU_END / TAU_START) ** (1 / iters))
    with pytest.raises(ValueError):
        default_tau(0.0)


def test_default_tau_schedules_are_bit_exact():
    """both fits' default schedules equal their closed forms to the last bit: the depth fit's d TAU_END (TAU_START /
    TAU_END)^x and the contour fit's end (start / end)^x, x = (iters - i) / max(iters, 1)"""
    from nope_b200 import contour_refine as cr, depth_refine as dr
    for iters in range(13):
        x = (iters - np.arange(iters + 1, dtype=np.float64)) / max(iters, 1)
        for d in (1e-3, 0.7, 80.0, 123.456, 2.0 * 97.3, 1e5):
            assert np.array_equal(dr.default_tau(d, iters), d * dr.TAU_END * (dr.TAU_START / dr.TAU_END) ** x)
        for start, end in ((cr.TAU_START, cr.TAU_END), (0.3, 0.05), (0.5, 0.5), (0.01, 0.2)):
            assert np.array_equal(cr.default_tau(iters, start, end), end * (start / end) ** x)
        assert np.array_equal(cr.default_tau(iters), cr.TAU_END * (cr.TAU_START / cr.TAU_END) ** x)


# ------------------------------------------------------------------ argument errors
def test_argument_errors():
    from nope_b200 import _lib
    from nope_b200.depth_refine import refine_pose_depth
    from nope_b200.vsd import Mesh
    v, f = ro.box()
    mesh = Mesh(v, f, device="cpu")
    F = 2
    R, t = np.eye(3)[None].repeat(F, 0), np.tile([0.0, 0.0, 300.0], (F, 1))
    S = np.zeros((F, 8, 10))
    ok = dict(mesh=mesh, R=R, t=t, K=K4, depth=S)
    with pytest.raises(_lib.NopeError):                          # no CPU fallback
        refine_pose_depth(**ok)
    for bad in (dict(mesh=(v, f)), dict(R=R[:, :2]), dict(R=R.astype(np.int32)), dict(t=t[:, :2]), dict(t=t[:1]),
                dict(depth=S[:1]), dict(depth=S.astype(np.uint16)), dict(masks=np.ones((F, 8, 9), np.uint8)),
                dict(masks=np.ones((F, 8, 10), np.float32)), dict(iters=-1), dict(iters=1.5), dict(iters=2000),
                dict(tau=[1.0, 2.0]), dict(tau=0.0), dict(tau=np.inf), dict(znear=0.0), dict(K=np.ones((3, 4)))):
        with pytest.raises(ValueError):
            refine_pose_depth(**{**ok, **bad})
    with pytest.raises(ValueError):
        refine_pose_depth(**ok, iters=2, tau=[3.0, 2.0, -1.0])


def test_c_abi_refuses_bad_arguments():
    """every refusal happens before any CUDA call, so it holds without a GPU"""
    from nope_b200 import _lib
    lib = _lib.load()
    K = np.array([[150.0, 151.0, 48.0, 36.0]])
    tau = np.array([4.0, 2.0, 1.0])

    def call(F=1, P=1, H=8, W=8, iters=2, znear=0.05, k=K, null=None, V=3, NF=1, rho=50.0, tv=tau):
        args = [1, V, 1, NF, 1, 1, 1, None, k.ctypes.data, F, P, H, W, rho, tv.ctypes.data, iters, znear, 1, 1, 1, 1,
                None, None]
        if null is not None:
            args[null] = None
        return lib.nope_refine_depth(*args)
    for kw in (dict(F=0), dict(F=65536), dict(P=0), dict(P=65536), dict(H=0), dict(W=8193), dict(iters=-1),
               dict(iters=1025), dict(znear=0.0), dict(znear=math.inf), dict(rho=0.0), dict(rho=-1.0),
               dict(rho=math.nan), dict(tv=tau * [1, 1, 0]), dict(tv=tau * [1, -1, 1]), dict(tv=tau * [np.nan, 1, 1]),
               dict(k=K * [np.nan, 1, 1, 1]), dict(k=K * [1, 0, 1, 1]), dict(k=K * [1, 1, np.inf, 1]), dict(V=0),
               dict(NF=0), dict(null=0), dict(null=2), dict(null=4), dict(null=5), dict(null=6), dict(null=8),
               dict(null=14), dict(null=17), dict(null=18), dict(null=19), dict(null=20)):
        with pytest.raises(_lib.NopeError):
            _lib.check(call(**kw))
