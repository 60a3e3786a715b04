"""CPU: the translation fit of DESIGN.md section 18.  The update on hand-built statistics (a shifted silhouette moves
only x and y, a scaled one only the distance), `initial_translation` against the numpy oracle, argument errors, and
the oracle end to end on small frames rendered by oracle/render_oracle, where it converges to the true translation."""
import math

import numpy as np
import pytest
import torch

import translation_oracle as to
from oracle import render_oracle as ro

K4 = np.array([150.0, 151.0, 48.2, 35.9])                    # the 96 x 72 intrinsics of tests/test_bop_gpu.py
KP = np.array([1075.65091572, 1073.90347929, 360.0, 270.0])   # Primesense, 720 x 540


def _box(r0, r1, c0, c1):
    return (1, 0, r0, r1, c0, c1)


# ------------------------------------------------------------------ the update on hand-built statistics
@pytest.mark.parametrize("du,dv", [(7, 0), (0, -5), (-12, 9), (1, 1)])
def test_shifted_silhouette_moves_only_x_and_y(du, dv):
    t = np.array([23.0, -41.0, 612.0])
    msk = _box(200, 259, 300, 379)
    sil = _box(200 + dv, 259 + dv, 300 + du, 379 + du)
    t1 = to.update(t, sil, msk, KP)
    assert t1[2] == t[2]
    assert abs(t1[0] - (t[0] - du * t[2] / KP[0])) <= 1e-12 * t[2]
    assert abs(t1[1] - (t[1] - dv * t[2] / KP[1])) <= 1e-12 * t[2]


@pytest.mark.parametrize("sigma", [0.5, 2.0, 1.25])
def test_scaled_silhouette_moves_only_z(sigma):
    """a silhouette that is the mask scaled by sigma about the projected origin: z -> z sigma.  With the origin on the
    optical axis x and y stay 0; elsewhere the origin keeps its projection (x / z is unchanged)."""
    z = 800.0
    M = np.array([240.0, 320.0, 400.0, 480.0])                  # mask box edges [r_lo, r_hi), [c_lo, c_hi) in px
    for x, y, cx, cy in ((0.0, 0.0, 360.0, 268.0), (40.0, -32.0, 350.0, 260.0)):
        K = np.array([1000.0, 1000.0, cx, cy])
        pu, pv = K[0] * x / z + cx, K[1] * y / z + cy
        assert pu == round(pu) and pv == round(pv)
        S = np.array([pv + (M[0] - pv) * sigma, pv + (M[1] - pv) * sigma, pu + (M[2] - pu) * sigma,
                      pu + (M[3] - pu) * sigma])
        assert (S == np.round(S)).all()
        msk = _box(int(M[0]), int(M[1]) - 1, int(M[2]), int(M[3]) - 1)
        sil = _box(int(S[0]), int(S[1]) - 1, int(S[2]), int(S[3]) - 1)
        t1 = to.update(np.array([x, y, z]), sil, msk, K)
        assert t1[2] == z * sigma
        if x == 0.0:
            assert t1[0] == 0.0 and t1[1] == 0.0
        assert abs(t1[0] / t1[2] - x / z) < 1e-15 and abs(t1[1] / t1[2] - y / z) < 1e-15


def test_empty_silhouette_or_mask_keeps_t():
    t = np.array([1.0, 2.0, 300.0])
    empty = (0, 0, 2 ** 31 - 1, -1, 2 ** 31 - 1, -1)
    assert np.array_equal(to.update(t, empty, _box(1, 5, 1, 5), K4), t)
    assert np.array_equal(to.update(t, _box(1, 5, 1, 5), empty, K4), t)


# ------------------------------------------------------------------ initial_translation
def _masks(seed, F=6, H=72, W=96):
    rng = np.random.default_rng(seed)
    m = np.zeros((F, H, W), dtype=np.uint8)
    for f in range(F):
        r0, c0 = rng.integers(0, H - 10), rng.integers(0, W - 10)
        m[f, r0:r0 + rng.integers(1, 10), c0:c0 + rng.integers(1, 10)] = rng.integers(1, 256)
        m[f] *= rng.random((H, W)) < 0.8                          # holes do not change the box
    m[0, 0, 0] = 7                                               # a box touching the corner
    return m


def test_initial_translation_matches_oracle():
    from nope_b200.translation import initial_translation, mask_box
    m = _masks(0)
    K = np.stack([K4 * [1, 1 + 0.01 * f, 1, 1] for f in range(len(m))])
    d = np.linspace(50.0, 180.0, len(m))
    t = initial_translation(torch.from_numpy(m), torch.from_numpy(K), torch.from_numpy(d)).numpy()
    for f in range(len(m)):
        assert np.array_equal(t[f], to.initial_translation(m[f], K[f], d[f])), f
    n, r0, r1, c0, c1 = (x.numpy() for x in mask_box(torch.from_numpy(m)))
    for f in range(len(m)):
        assert (n[f], r0[f], r1[f], c0[f], c1[f]) == tuple(np.array(to.stats(m[f] != 0))[[0, 2, 3, 4, 5]])
    # one K, one diameter, bool masks, [3, 3] intrinsics: the same numbers
    K33 = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1.0]])
    t1 = initial_translation(torch.from_numpy(m != 0), K33, 120.0).numpy()
    for f in range(len(m)):
        assert np.array_equal(t1[f], to.initial_translation(m[f], K4, 120.0))


def test_initial_translation_of_an_empty_mask_is_nan():
    from nope_b200.translation import initial_translation
    m = _masks(1)
    m[2] = 0
    t = initial_translation(m, K4, 100.0).numpy()
    assert np.isnan(t[2]).all() and np.isfinite(np.delete(t, 2, axis=0)).all()
    assert np.isnan(to.initial_translation(m[2], K4, 100.0)).all()


def test_initial_translation_of_a_rendered_object():
    """a sphere of diameter d seen head-on: its box is about d fx / z wide, so z0 is close to z"""
    v, f = ro.sphere(40.0, 2)
    t_true = np.array([8.0, -5.0, 400.0])
    d = ro.render(v, f, to.pose(np.eye(3), t_true), K4, (72, 96))[0].numpy()
    t0 = to.initial_translation(d > 0, K4, 80.0)
    assert abs(t0[2] - 400.0) < 0.1 * 400.0
    assert abs(t0[0] - 8.0) < 3.0 and abs(t0[1] + 5.0) < 3.0


# ------------------------------------------------------------------ argument errors
def test_argument_errors():
    from nope_b200 import _lib
    from nope_b200.translation import estimate_translation, initial_translation
    from nope_b200.vsd import Mesh
    v, f = ro.box()
    m = _masks(2)
    with pytest.raises(_lib.NopeError):                          # no CPU fallback
        estimate_translation(Mesh(v, f, device="cpu"), np.eye(3)[None].repeat(6, 0), K4, m, diameter=80.0)
    with pytest.raises(ValueError):
        estimate_translation((v, f), np.eye(3)[None].repeat(6, 0), K4, m, diameter=80.0)
    with pytest.raises(ValueError):
        initial_translation(m.astype(np.float32), K4, 80.0)
    with pytest.raises(ValueError):
        initial_translation(m, np.ones((2, 4)), 80.0)
    with pytest.raises(ValueError):
        initial_translation(m, K4, np.ones(4))
    with pytest.raises(ValueError):
        initial_translation(np.zeros((1, 0, 5), dtype=np.uint8), K4, 80.0)


def test_c_abi_refuses_bad_arguments():
    """every refusal happens before any CUDA call, so it holds without a GPU"""
    from nope_b200 import _lib
    lib = _lib.load()
    K = np.array([[150.0, 151.0, 48.0, 36.0]])

    def call(F=1, P=1, H=8, W=8, iters=2, znear=0.05, k=K, null=None, V=3, NF=1):
        args = [1, V, 1, NF, 1, 1, 1, k.ctypes.data, F, P, H, W, znear, iters, 1, 1, 1, None, None]
        if null is not None:
            args[null] = None
        return lib.nope_fit_translation_occluded(*args[:7], None, *args[7:])     # occluders NULL
    for kw in (dict(F=0), dict(F=65536), dict(P=0), dict(P=65536), dict(H=0), dict(W=8193), dict(iters=-1),
               dict(znear=0.0), dict(znear=-1.0), dict(znear=math.inf), dict(k=K * [np.nan, 1, 1, 1]),
               dict(k=K * [1, 0, 1, 1]), dict(k=K * [1, 1, np.inf, 1]), dict(V=0), dict(NF=0), dict(null=0),
               dict(null=2), dict(null=4), dict(null=5), dict(null=6), dict(null=7), dict(null=14), dict(null=15),
               dict(null=16)):
        with pytest.raises(_lib.NopeError):
            _lib.check(call(**kw))


# ------------------------------------------------------------------ the oracle end to end
@pytest.mark.parametrize("mesh", ["box", "sphere", "soup"])
def test_oracle_converges_to_the_true_translation(mesh):
    v, f = {"box": ro.box, "sphere": lambda: ro.sphere(40.0, 1), "soup": lambda: ro.soup(24, seed=3)}[mesh]()
    diameter = float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))
    rng = np.random.default_rng(5)
    render = to.cpu_renderer(v, f, K4, (72, 96))
    for _ in range(2):
        R = ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)
        t_true = np.array([rng.uniform(-15, 15), rng.uniform(-10, 10), rng.uniform(300, 420)])
        mask = render(R, t_true) > 0
        t0 = to.initial_translation(mask, K4, diameter)
        t, iou, sil = to.fit(render, R, t0, mask, K4, 4)
        msk = to.stats(mask)
        bound = 2 * t_true[2] / math.sqrt((msk[5] - msk[4] + 1) * (msk[3] - msk[2] + 1))
        assert abs(t[2] - t_true[2]) <= bound, (t, t_true, bound)
        u, w = K4[0] * t[0] / t[2] + K4[2], K4[1] * t[1] / t[2] + K4[3]
        ut, wt = K4[0] * t_true[0] / t_true[2] + K4[2], K4[1] * t_true[1] / t_true[2] + K4[3]
        assert math.hypot(u - ut, w - wt) <= 1.0, (u, w, ut, wt)
        assert iou > 0.7 and sil[0] > 0                      # thin soup triangles at 96 x 72 lose most to 1 px
        # from the true translation the fit stays there
        t, iou, _ = to.fit(render, R, t_true, mask, K4, 2)
        assert np.abs(t - t_true).max() <= 1e-6 and iou == 1.0
