"""GPU: the pose fits under occlusion (DESIGN.md section 24).  Scenes from the depth rasterizer: a target (box,
icosphere) at 400 - 1200 mm in the 720 x 540 Primesense frame, a sphere placed nearer so that it hides about 20, 40 or
60 % of the target's silhouette, M = the target's pixels in front of the occluder, O = the occluder's silhouette.
Both fits against the numpy oracle bit for bit; the occluded entry points without occluders against the plain ones;
the true pose as a fixed point; accuracy with and without O; batch independence and no host synchronisation; and the
PoseConditional entry points, predict_pose_frames(occluders="detections") included."""
import math
import types

import numpy as np
import pytest
import torch

import contour_refine_oracle as cro
import occlusion_fit_oracle as ofo
import translation_oracle as to
from oracle import render_oracle as ro
from test_depth_refine_gpu import _angle, _perturb

pytestmark = pytest.mark.gpu

K4 = np.array([1075.65091572, 1073.90347929, 360.0, 270.0])    # Primesense
H, W = 540, 720
MESHES = {"box": lambda: ro.box(), "sphere": lambda: ro.sphere(40.0, 2)}
OCC_RADIUS = 25.0                                             # mm, the occluding sphere
TAUS = np.geomspace(0.15, 0.02, 7)


def _mesh(name):
    from nope_b200.vsd import Mesh
    v, f = MESHES[name]()
    return Mesh(v, f), float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))


def _occluder():
    from nope_b200.vsd import Mesh
    return Mesh(*ro.sphere(OCC_RADIUS, 2))


def _render(mesh, R, t, K=K4):
    from nope_b200.vsd import render_depth
    return render_depth(mesh, torch.from_numpy(to.pose(R, t)), K, (H, W))[0]


def _inside(m):
    rows, cols = m.any(1).nonzero(), m.any(0).nonzero()
    return len(rows) > 0 and rows.min() > 0 and cols.min() > 0 and rows.max() < H - 1 and cols.max() < W - 1


def occluded_scene(mesh, seed, F, cover, behind=False, K=K4):
    """F frames: a true pose each, the target's visible mask M and the occluders O (uint8 [F, H, W] on the GPU), and
    the coverage achieved: a sphere of radius OCC_RADIUS about as large in the image as the target and at least 120 mm
    nearer the camera,
    moved from the target's box centre along a seeded direction until it hides `cover` of the target's silhouette
    (bisection, within 0.04).  With `behind`, O also holds a box 150 mm behind the target, beside it.
    -> (R_true [F, 3, 3], t_true [F, 3], M, O, coverage [F], S the target's full silhouettes, t_occ [F, 3] the
    sphere's centres)"""
    rng = np.random.default_rng(seed)
    occ = _occluder()
    fx, fy, cx, cy = K
    back = None
    if behind:
        from nope_b200.vsd import Mesh
        back = Mesh(*ro.box(80.0, 60.0, 10.0))
    Rt, tt, Ms, Os, cov, Ss, To = [], [], [], [], [], [], []
    while len(Rt) < F:
        R = ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)
        z = rng.uniform(400.0, 1200.0)
        t = np.array([rng.uniform(-0.15, 0.15) * z, rng.uniform(-0.15, 0.15) * z, z])
        D = _render(mesh, R, t, K)
        S = D > 0
        if not _inside(S):
            continue
        n, _, r0, r1, c0, c1 = to.stats(S.cpu().numpy())
        rs = math.sqrt(n / math.pi)
        zo = min(fx * OCC_RADIUS / rs, z - 120.0)                 # in front of the target's 40 mm radius
        a = rng.uniform(0, 2 * math.pi)
        u0, v0 = (c0 + c1 + 1) / 2, (r0 + r1 + 1) / 2

        def place(d):
            u, v = u0 + d * math.cos(a), v0 + d * math.sin(a)
            to_ = np.array([(u - cx) * zo / fx, (v - cy) * zo / fy, zo])
            Do = _render(occ, np.eye(3), to_, K)
            return Do, float((S & (Do > 0) & (Do < D)).sum()) / n, to_
        lo, hi = 0.0, 3.0 * rs
        for _ in range(16):
            mid = 0.5 * (lo + hi)
            if place(mid)[1] > cover:
                lo = mid
            else:
                hi = mid
        Do, c, to_ = place(0.5 * (lo + hi))
        if abs(c - cover) > 0.04:
            continue
        assert bool((~((Do > 0) & S) | (Do < D)).all())             # the sphere is in front wherever it overlaps
        M = S & ~((Do > 0) & (Do < D))
        O = Do > 0
        if behind:
            tb = t + np.array([1.4 * rs * z / fx, 0.0, 150.0])
            Db = _render(back, np.eye(3), tb, K)
            assert bool((~((Db > 0) & S) | (D < Db)).all())
            O = O | (Db > 0)
        Rt.append(R), tt.append(t), Ms.append(M.to(torch.uint8)), Os.append(O.to(torch.uint8)), cov.append(c)
        Ss.append(S), To.append(to_)
    return (np.stack(Rt), np.stack(tt), torch.stack(Ms), torch.stack(Os), np.array(cov), torch.stack(Ss),
            np.stack(To))


# ------------------------------------------------------------------ kernels = oracle
@pytest.mark.parametrize("name", ["box", "sphere"])
@pytest.mark.parametrize("P", [1, 5])
def test_translation_equals_oracle(name, P):
    from nope_b200.translation import estimate_translation, initial_translation
    mesh, diameter = _mesh(name)
    F = 2
    K = np.stack([K4, K4 * [1.0, 1.001, 1.02, 0.98]])
    R_true, _, M, O, *_ = occluded_scene(mesh, 11 + P, F, 0.4, K=K4)
    rng = np.random.default_rng(P)
    R = np.stack([np.stack([R_true[f]] + [ro.look_pose(*rng.uniform(-3, 3, 3))[:3, :3].astype(np.float64)
                                          for _ in range(P - 1)]) for f in range(F)])
    t0 = initial_translation(M, K, diameter)
    got = [estimate_translation(mesh, R, K, M, t_init=t0, iters=i, return_stats=True, occluders=O) for i in range(7)]
    got = [tuple(x.cpu().numpy() for x in g) for g in got]
    Mh, Oh = M.cpu().numpy(), O.cpu().numpy()
    for f in range(F):
        msk = to.stats(ofo.visible(Mh[f], Oh[f]))
        for p in range(P):
            t = t0[f].cpu().numpy()
            for i in range(7):
                sil = ofo.translation_stats(_render(mesh, R[f, p], t, K[f]).cpu().numpy(), Mh[f], Oh[f])
                assert tuple(got[i][2][f, p]) == sil, (f, p, i)
                assert np.array_equal(got[i][0][f, p], t), (f, p, i, got[i][0][f, p], t)
                assert got[i][1][f, p] == to.iou(sil, msk), (f, p, i)
                t = to.update(t, sil, msk, K[f])


@pytest.mark.parametrize("name", ["box", "sphere"])
@pytest.mark.parametrize("P", [1, 5])
def test_contour_equals_oracle(name, P):
    from nope_b200.contour_refine import refine_pose_contour
    mesh, _ = _mesh(name)
    F = 2
    K = np.stack([K4, K4 * [1.0, 1.001, 1.02, 0.98]])
    R_true, t_true, M, O, *_ = occluded_scene(mesh, 41 + P, F, 0.4)
    rng = np.random.default_rng(P)
    st = [[_perturb(rng, R_true[f], t_true[f]) for _ in range(P)] for f in range(F)]
    R0 = np.array([[s[0] for s in row] for row in st])
    t0 = np.array([[s[1] for s in row] for row in st])
    got = [refine_pose_contour(mesh, R0, t0, K, M, iters=i, tau=TAUS[:i + 1], return_sums=True, occluders=O)
           for i in range(7)]
    got = [(g[0].cpu().numpy(), g[1].cpu().numpy(), torch.stack([g[2][k] for k in ("n_in", "n_contour", "rms",
           "iou")], -1).cpu().numpy(), g[3].cpu().numpy()) for g in got]
    Mh, Oh = M.cpu().numpy(), O.cpu().numpy()
    rho = mesh.radius
    for f in range(F):
        mv = ofo.visible(Mh[f], Oh[f])
        phi, s = cro.sdf(mv), cro.box_size(mv)
        for p in range(P):
            R, t = R0[f, p], t0[f, p]
            for i in range(7):
                D = _render(mesh, R, t, K[f]).cpu().numpy()
                tau = TAUS[i] * s
                sums, nc = ofo.accumulate(D, phi, K[f], t, tau, rho, Oh[f])
                assert np.array_equal(got[i][3][f, p], sums), (f, p, i, got[i][3][f, p] - sums)
                assert np.array_equal(got[i][0][f, p], R) and np.array_equal(got[i][1][f, p], t), (f, p, i)
                nin = float(sums[-1])
                with np.errstate(invalid="ignore", divide="ignore"):
                    rms = tau * np.sqrt(np.float64(cro.dro.unfix(sums[-2])) / np.float64(nin))
                fit = np.array([nin, float(nc), rms, ofo.iou(D, Mh[f], Oh[f])])
                assert np.array_equal(got[i][2][f, p], fit, equal_nan=True), (f, p, i, got[i][2][f, p], fit)
                R, t = cro.solve(sums, R, t, tau, K[f], rho)
        assert got[6][3][f, :, -1].max() > 20                         # pairs were found


def test_workspaces_hold_the_final_render():
    from nope_b200 import _lib
    from nope_b200.vsd import _stream
    mesh, diameter = _mesh("box")
    R_true, t_true, M, O, *_ = occluded_scene(mesh, 3, 2, 0.3)
    Rd = torch.from_numpy(R_true).cuda().contiguous()
    td = torch.from_numpy(t_true + [3.0, -2.0, 15.0]).cuda().contiguous()
    K = np.repeat(K4[None], 2, axis=0)
    depth = torch.empty((2, H, W), device="cuda")
    f64 = dict(device="cuda", dtype=torch.float64)
    t, iou = torch.empty((2, 3), **f64), torch.empty(2, **f64)
    _lib.check(_lib.load().nope_fit_translation_occluded(
        _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
        _lib.ptr(td), _lib.ptr(M), _lib.ptr(O), K.ctypes.data, 2, 1, H, W, 0.05, 3, _lib.ptr(depth), _lib.ptr(t),
        _lib.ptr(iou), None, _stream(torch.device("cuda"))))
    for f in range(2):
        assert torch.equal(depth[f], _render(mesh, R_true[f], t[f].cpu().numpy()))
    R, fit = torch.empty((2, 3, 3), **f64), torch.empty((2, 4), **f64)
    tau = TAUS[:4].copy()
    _lib.check(_lib.load().nope_refine_contour_occluded(
        _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(Rd),
        _lib.ptr(td), _lib.ptr(M), _lib.ptr(O), K.ctypes.data, 2, 1, H, W, mesh.radius, tau.ctypes.data, 3, 0.05,
        _lib.ptr(depth), _lib.ptr(R), _lib.ptr(t), _lib.ptr(fit), None, _stream(torch.device("cuda"))))
    for f in range(2):
        assert torch.equal(depth[f], _render(mesh, R[f].cpu().numpy(), t[f].cpu().numpy()))


# ------------------------------------------------------------------ without occluders: the plain fits, bit for bit
def test_no_or_zero_occluders_are_the_plain_fits():
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import estimate_translation
    mesh, diameter = _mesh("box")
    R_true, t_true, M, O, *_ = occluded_scene(mesh, 5, 3, 0.4)
    rng = np.random.default_rng(2)
    st = [[_perturb(rng, R_true[f], t_true[f]) for _ in range(4)] for f in range(3)]
    R0 = np.array([[s[0] for s in row] for row in st])
    t0 = np.array([[s[1] for s in row] for row in st])
    zero = torch.zeros_like(O)
    a = estimate_translation(mesh, R0, K4, M, diameter=diameter, return_stats=True)
    for occ in (None, zero, zero.bool()):
        b = estimate_translation(mesh, R0, K4, M, diameter=diameter, return_stats=True, occluders=occ)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = refine_pose_contour(mesh, R0, t0, K4, M, return_sums=True)
    for occ in (None, zero):
        b = refine_pose_contour(mesh, R0, t0, K4, M, return_sums=True, occluders=occ)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])
        assert all(torch.equal(a[2][k], b[2][k]) for k in a[2])
    # and O changes the result
    b = refine_pose_contour(mesh, R0, t0, K4, M, return_sums=True, occluders=O)
    assert not torch.equal(a[1], b[1])
    with pytest.raises(ValueError):
        estimate_translation(mesh, R0, K4, M, diameter=diameter, occluders=O[:2])
    with pytest.raises(ValueError):
        refine_pose_contour(mesh, R0, t0, K4, M, occluders=O[:, :, :-1])


# ------------------------------------------------------------------ the true pose is a fixed point
@pytest.mark.parametrize("name", ["box", "sphere"])
@pytest.mark.parametrize("behind", [False, True])
def test_the_true_pose_is_a_fixed_point(name, behind):
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import DEFAULT_ITERS, estimate_translation
    mesh, _ = _mesh(name)
    for cover in (0.2, 0.4, 0.6):
        R_true, t_true, M, O, *_ = occluded_scene(mesh, 7, 4, cover, behind=behind)
        t, iou = estimate_translation(mesh, R_true, K4, M, t_init=t_true, iters=DEFAULT_ITERS, occluders=O)
        assert np.abs(t[:, 0].cpu().numpy() - t_true).max() <= 1e-6 and iou.min().item() >= 0.999, (cover, iou)
        R, t, fit = refine_pose_contour(mesh, R_true, t_true, K4, M, occluders=O)
        assert np.array_equal(R[:, 0].cpu().numpy(), R_true) and np.array_equal(t[:, 0].cpu().numpy(), t_true)
        assert (fit["iou"] >= 0.999).all() and (fit["rms"] == 0).all() and (fit["n_in"] > 20).all(), (cover, fit)


# ------------------------------------------------------------------ accuracy
# Gates with O, from DESIGN.md section 24's table (32 scenes per mesh and level, seed 100; the test takes the first
# 16): (translation after the default 4 updates: median |dz| in box px, median reprojection px; contour: median
# |t - t_true| mm).  Measured: box 0.52 / 0.42 / 2.2, 0.38 / 0.38 / 2.5, 0.50 / 0.46 / 3.2 at 20 / 40 / 60 %;
# icosphere 0.25 / 0.39 / 0.9, 0.33 / 0.34 / 1.1, 0.35 / 0.34 / 1.2.  Without O the medians are 2.7 - 9.0 px and
# 3.8 - 6.6 mm.
GATES = {("box", 0.2): (1.2, 1.0, 4.0), ("box", 0.4): (1.2, 1.0, 4.5), ("box", 0.6): (1.2, 1.0, 5.5),
         ("sphere", 0.2): (0.8, 0.8, 2.0), ("sphere", 0.4): (0.8, 0.8, 2.2), ("sphere", 0.6): (0.8, 0.8, 2.5)}


def accuracy(mesh, diameter, name, cover, n, seed=100, iters=None):
    """-> dict of per-scene errors with ("O") and without ("no O") occluders: translation fit from
    initial_translation at the true rotation ("dz_px", "reproj_px"), contour fit from a start 2.5 - 5 deg and 5 - 10 mm
    off ("t_mm", "r_deg")"""
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import DEFAULT_ITERS, estimate_translation
    R_true, t_true, M, O, _, S, _ = occluded_scene(mesh, seed, n, cover)
    box = np.array([math.sqrt((s[5] - s[4] + 1) * (s[3] - s[2] + 1)) for s in (to.stats(x) for x in S.cpu().numpy())])
    rng = np.random.default_rng(seed + 1)
    st = [_perturb(rng, R_true[f], t_true[f]) for f in range(n)]
    R0, t0 = np.array([s[0] for s in st]), np.array([s[1] for s in st])
    out = {}
    for key, occ in (("O", O), ("no O", None)):
        t, _ = estimate_translation(mesh, R_true, K4, M, diameter=diameter,
                                    iters=DEFAULT_ITERS if iters is None else iters, occluders=occ)
        t = t[:, 0].cpu().numpy()
        u = K4[:2] * t[:, :2] / t[:, 2:] + K4[2:]
        ut = K4[:2] * t_true[:, :2] / t_true[:, 2:] + K4[2:]
        R, tc, _ = refine_pose_contour(mesh, R0, t0, K4, M, occluders=occ)
        R, tc = R[:, 0].cpu().numpy(), tc[:, 0].cpu().numpy()
        out[key] = {"dz_px": np.abs(t[:, 2] - t_true[:, 2]) * box / t_true[:, 2],
                    "reproj_px": np.linalg.norm(u - ut, axis=1),
                    "t_mm": np.linalg.norm(tc - t_true, axis=1),
                    "r_deg": np.array([_angle(R[f], R_true[f]) for f in range(n)])}
    return out


@pytest.mark.parametrize("name", ["box", "sphere"])
@pytest.mark.parametrize("cover", [0.2, 0.4, 0.6])
def test_accuracy_with_and_without_occluders(name, cover):
    mesh, diameter = _mesh(name)
    e = accuracy(mesh, diameter, name, cover, 16)
    med = {k: {m: float(np.median(v)) for m, v in e[k].items()} for k in e}
    print(f"{name} {cover:.0%}: with O {med['O']}; without O {med['no O']}")
    dz, rp, tmm = GATES[name, cover]
    assert med["O"]["dz_px"] <= dz and med["O"]["reproj_px"] <= rp and med["O"]["t_mm"] <= tmm, med
    assert med["O"]["reproj_px"] < med["no O"]["reproj_px"] and med["O"]["t_mm"] < med["no O"]["t_mm"], med


# ------------------------------------------------------------------ batch independence, synchronisation
def test_batch_independence():
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import estimate_translation
    mesh, diameter = _mesh("box")
    R_true, t_true, M, O, *_ = occluded_scene(mesh, 21, 3, 0.4)
    K = np.stack([K4 * [1, 1, 1 + 0.002 * f, 1] for f in range(3)])
    rng = np.random.default_rng(3)
    st = [[_perturb(rng, R_true[f], t_true[f]) for _ in range(4)] for f in range(3)]
    R0 = np.array([[s[0] for s in row] for row in st])
    t0 = np.array([[s[1] for s in row] for row in st])
    t, iou = estimate_translation(mesh, R0, K, M, diameter=diameter, occluders=O)
    R, tc, fit = refine_pose_contour(mesh, R0, t0, K, M, occluders=O)
    perm = [2, 0, 3, 1]
    for f in range(3):
        a, b = estimate_translation(mesh, R0[f:f + 1], K[f:f + 1], M[f:f + 1], diameter=diameter,
                                    occluders=O[f])
        assert torch.equal(a, t[f:f + 1]) and torch.equal(b, iou[f:f + 1])
        a, b, c = refine_pose_contour(mesh, R0[f:f + 1], t0[f:f + 1], K[f:f + 1], M[f:f + 1], occluders=O[f:f + 1])
        assert torch.equal(a, R[f:f + 1]) and torch.equal(b, tc[f:f + 1])
        assert all(torch.equal(c[k], fit[k][f:f + 1]) for k in c)
    a, b = estimate_translation(mesh, R0[:, perm], K, M, diameter=diameter, occluders=O)
    assert torch.equal(a, t[:, perm]) and torch.equal(b, iou[:, perm])
    a, b, c = refine_pose_contour(mesh, R0[:, perm], t0[:, perm], K, M, occluders=O)
    assert torch.equal(a, R[:, perm]) and torch.equal(b, tc[:, perm])


def test_no_host_synchronisation():
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.crop import detection_occluders
    from nope_b200.translation import estimate_translation
    mesh, diameter = _mesh("box")
    R_true, t_true, M, O, *_ = occluded_scene(mesh, 9, 2, 0.4)
    Rd, td = torch.from_numpy(R_true).cuda(), torch.from_numpy(t_true).cuda()
    K = np.repeat(K4[None], 2, axis=0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = estimate_translation(mesh, Rd, K, M, diameter=diameter, occluders=O)
        b = refine_pose_contour(mesh, Rd, td, K, M.bool(), occluders=O.bool())
        c = detection_occluders(M, torch.tensor([0, 0]), num_frames=1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a[0], estimate_translation(mesh, R_true, K, M.cpu(), diameter=diameter, occluders=O.cpu())[0])
    assert torch.isfinite(b[1]).all()
    assert torch.equal(c.cpu(), torch.from_numpy(ofo.detection_occluders(M.cpu().numpy(), [0, 0])))


# ------------------------------------------------------------------ PoseConditional
def _two_object_batch():
    """four rows, objects 91 (box) and 92 (sphere) interleaved, each with its own occluders"""
    boxm, boxd = _mesh("box")
    sphm, sphd = _mesh("sphere")
    Rb, tb, Mb, Ob, *_ = occluded_scene(boxm, 31, 2, 0.4)
    Rs, ts, Ms, Os, *_ = occluded_scene(sphm, 32, 2, 0.4)
    order = [0, 2, 1, 3]                                      # box, sphere, box, sphere
    R = np.concatenate([Rb, Rs])[order]
    t = np.concatenate([tb, ts])[order]
    M, O = torch.cat([Mb, Ms])[order], torch.cat([Ob, Os])[order]
    K = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]])
    batch = {"intrinsic": torch.from_numpy(K)[None].expand(4, 3, 3), "obj_id": torch.tensor([91, 92, 91, 92])}
    return {91: (boxm, boxd), 92: (sphm, sphd)}, batch, R, t, M, O


def _with_objects(model, meshes):
    from nope_b200 import bop
    for i, (mesh, d) in meshes.items():
        info = {"diameter": d, "symmetries_discrete": [], "symmetries_continuous": []}
        model.tless_cad[i] = mesh
        model.bop_models[i] = {"diameter": d, "symmetries": bop.symmetry_transformations(info), "info": info}
    return model


def test_pose_conditional_routes_occluders_per_object():
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.model import PoseConditional
    from nope_b200.translation import estimate_translation
    meshes, batch, R, t, M, O = _two_object_batch()
    model = _with_objects(PoseConditional(types.SimpleNamespace(device=torch.device("cuda", 0))), meshes)
    rng = np.random.default_rng(8)
    st = [[_perturb(rng, R[b], t[b]) for _ in range(2)] for b in range(4)]
    R0 = np.array([[s[0] for s in row] for row in st])
    t0 = np.array([[s[1] for s in row] for row in st])
    ta, ia = model.estimate_translation(batch, R0, M, occluders=O)
    Ra, tc, ic = model.refine_contour(batch, R0, t0, M, occluders=O)
    K = batch["intrinsic"][0].numpy()
    for b, i in enumerate([91, 92, 91, 92]):
        mesh, d = meshes[i]
        x, y = estimate_translation(mesh, R0[b:b + 1], K, M[b:b + 1], diameter=d, occluders=O[b:b + 1])
        assert torch.equal(ta[b], x[0]) and torch.equal(ia[b], y[0])
        x, y, z = refine_pose_contour(mesh, R0[b:b + 1], t0[b:b + 1], K, M[b:b + 1], occluders=O[b:b + 1])
        assert torch.equal(Ra[b], x[0]) and torch.equal(tc[b], y[0]) and torch.equal(ic[b], z["iou"][0])
    plain = model.estimate_translation(batch, R0, M)
    assert all(torch.equal(x, y) for x, y in zip(plain, model.estimate_translation(batch, R0, M, occluders=None)))
    assert not torch.equal(plain[0], ta)
    with pytest.raises(ValueError):
        model.refine_contour(batch, R0, t0, M, occluders=O[:3])


def _two_detections():
    """one frame, two detections: a box, and a sphere in front of it hiding about 40 % of it
    -> (meshes, ids, R [2, 3, 3], t [2, 3], masks uint8 0 / 255 [2, H, W], frames [1, H, W, 3], frame_idx)"""
    boxm, boxd = _mesh("box")
    R, t, _, _, _, _, to_ = occluded_scene(boxm, 51, 1, 0.4)
    occ = _occluder()
    to_ = to_[0]
    Do = _render(occ, np.eye(3), to_)
    D = _render(boxm, R[0], t[0])
    mask_box = ((D > 0) & ~((Do > 0) & (Do < D))).to(torch.uint8) * 255
    mask_sph = (Do > 0).to(torch.uint8) * 255
    masks = torch.stack([mask_box, mask_sph])
    frames = (masks[0] | masks[1])[None, ..., None].expand(1, H, W, 3).contiguous()
    meshes = {91: (boxm, boxd), 93: (occ, 2 * OCC_RADIUS)}
    return meshes, [91, 93], np.stack([R[0], np.eye(3)]), np.stack([t[0], to_]), masks, frames, torch.tensor([0, 0])


def test_predict_pose_frames_with_detection_occluders():
    """the search stubbed to the true crop rotation: with occluders="detections" the occluded box meets the
    translation gate, without them it is biased; the call equals estimate_translation with the detections'
    occluders by hand, and occluders=None equals the plain call"""
    from nope_b200 import translation
    from nope_b200.crop import detection_occluders, frame_crops, to_crop
    from nope_b200.model import PoseConditional
    meshes, ids, R, t, masks, frames, fi = _two_detections()
    model = _with_objects(PoseConditional(types.SimpleNamespace(device=torch.device("cuda", 0))), meshes)
    K3 = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]])
    d = np.array([meshes[i][1] for i in ids])
    _, t0, Rv, _ = frame_crops(frames, masks, K3, d, frame_idx=fi)
    k = 2
    R_crop = to_crop(torch.from_numpy(R).cuda()[:, None].expand(2, k, 3, 3), Rv)

    def search(query, reference, all_relativeR, template_poses, k, angles):
        zeros = torch.zeros((2, k), dtype=torch.int64, device="cuda")
        return R_crop, zeros, zeros, torch.zeros((2, angles, 4), device="cuda")
    model.predict_pose_inplane = search
    args = (frames, masks, K3, ids, torch.zeros(1, 3, 256, 256), torch.zeros(1, 4, 6), torch.zeros(4, 3, 3))
    out = model.predict_pose_frames(*args, k=k, frame_idx=fi, occluders="detections")
    plain = model.predict_pose_frames(*args, k=k, frame_idx=fi)
    none = model.predict_pose_frames(*args, k=k, frame_idx=fi, occluders=None)
    assert all(torch.equal(plain[key], none[key]) for key in plain)
    O = detection_occluders(masks, fi)
    m = masks != 0
    assert torch.equal(O[0].bool(), m[1] & ~m[0]) and torch.equal(O[1].bool(), m[0] & ~m[1])
    for b, i in enumerate(ids):
        tb, ib = translation.estimate_translation(meshes[i][0], out["R"][b:b + 1], K3, masks[b:b + 1],
                                                  t_init=t0[b:b + 1], occluders=O[b:b + 1])
        assert torch.equal(out["t"][b], tb[0]) and torch.equal(out["iou"][b], ib[0])
    e = lambda x: float(np.linalg.norm(K4[:2] * x[:2] / x[2] + K4[2:] - (K4[:2] * t[0, :2] / t[0, 2] + K4[2:])))  # noqa
    e_occ, e_plain = e(out["t"][0, 0].cpu().numpy()), e(plain["t"][0, 0].cpu().numpy())
    print(f"occluded detection: reprojection {e_occ:.2f} px with occluders, {e_plain:.2f} px without")
    assert e_occ <= 1.5 and e_plain > 2 * e_occ
    with pytest.raises(ValueError):
        model.predict_pose_frames(*args, k=k, frame_idx=fi, occluders="other detections")


def test_predict_pose_frames_detections_equals_the_chain(gpu_model):
    """with the seeded engine: predict_pose_frames(refine="contour", occluders="detections") equals the chain of its
    stages by hand, and it still synchronises only as its stages do, frame_crops once"""
    from nope_b200 import contour_refine, translation
    from nope_b200.crop import detection_occluders, frame_crops, to_camera
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from oracle import inputs
    from test_frame_pose_gpu import _syncs
    meshes, ids, _, _, masks, frames, fi = _two_detections()
    model = _with_objects(gpu_model, meshes)
    _, ref = inputs.make_images(seed=4, batch=1)
    ref, rel = ref.cuda(), synthetic_pose_batch(42, 1)[0].cuda()
    tp = torch.from_numpy(icosphere_object_rotations(0)).cuda()
    K3 = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]])
    args = (frames, masks, K3, ids, ref, rel, tp)
    out = model.predict_pose_frames(*args, angles=6, k=3, frame_idx=fi, refine="contour", occluders="detections")
    d = np.array([meshes[i][1] for i in ids])
    crops, t0, Rv, _ = frame_crops(frames, masks, K3, d, frame_idx=fi)
    R_crop, n, a, sim = model.predict_pose_inplane(crops, ref, rel, tp, k=3, angles=6)
    R = to_camera(R_crop, Rv)
    O = detection_occluders(masks, fi)
    for b, i in enumerate(ids):
        tt, _ = translation.estimate_translation(meshes[i][0], R[b:b + 1], K3, masks[b:b + 1], t_init=t0[b:b + 1],
                                                 occluders=O[b:b + 1])
        Rr, tr, fit = contour_refine.refine_pose_contour(meshes[i][0], R[b:b + 1], tt, K3, masks[b:b + 1],
                                                         occluders=O[b:b + 1])
        assert torch.equal(out["R"][b], Rr[0]) and torch.equal(out["t"][b], tr[0])
        assert torch.equal(out["iou"][b], fit["iou"][0])
    assert torch.equal(out["R_crop"], R_crop) and torch.equal(out["t0"], t0)
    _, n_occ = _syncs(lambda: model.predict_pose_frames(*args, angles=6, k=3, frame_idx=fi, refine="contour",
                                                        occluders="detections"))
    _, n_plain = _syncs(lambda: model.predict_pose_frames(*args, angles=6, k=3, frame_idx=fi, refine="contour"))
    print(f"syncs: with detection occluders {n_occ}, without {n_plain}")
    assert n_occ == n_plain
