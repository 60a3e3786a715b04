"""Seeded scenes shared by the pose-fit, frame, tracking, BOP and VSD tests and by the fit timing tools: the 720 x 540
Primesense camera, the test meshes, rotations and perturbations, depth renders, the depth-refine and occlusion scenes,
and a synthetic T-LESS batch.  Each helper draws from its rng in a fixed order: the tests' accuracy gates were tuned
on exactly these scenes."""
import math

import numpy as np
import torch

import translation_oracle as to
from oracle import render_oracle as ro

K4 = np.array([1075.65091572, 1073.90347929, 360.0, 270.0])    # Primesense, as tools/vsd_time.py
K3 = np.array([[K4[0], 0.0, K4[2]], [0.0, K4[1], K4[3]], [0.0, 0.0, 1.0]])
H, W = 540, 720
MESHES = {"box": lambda: ro.box(), "sphere": lambda: ro.sphere(40.0, 2), "soup": lambda: ro.soup(64, seed=1)}
FLIPS = [np.diag([1.0, -1.0, -1.0, 1.0]), np.diag([-1.0, 1.0, -1.0, 1.0]), np.diag([-1.0, -1.0, 1.0, 1.0])]
OCC_RADIUS = 25.0                                             # mm, the occluding sphere of occluded_scene


def make_mesh(name):
    """-> (the device Mesh of MESHES[name], its diameter: the largest distance between two vertices)"""
    from nope_b200.vsd import Mesh
    v, f = MESHES[name]()
    return Mesh(v, f), float(np.max(np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2)))


def rot(rng):
    return ro.look_pose(*rng.uniform(-math.pi, math.pi, 3))[:3, :3].astype(np.float64)


def rotvec(w):
    """rotation matrix of the rotation vector w (radians)"""
    w = np.asarray(w, dtype=np.float64)
    a = np.linalg.norm(w)
    if a == 0:
        return np.eye(3)
    k = w / a
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(a) * Kx + (1 - math.cos(a)) * Kx @ Kx


def angle(Ra, Rb):
    """the angle of Ra Rb^T in degrees, from the chord |Ra - Rb|_F = 2 sqrt(2) sin(angle / 2): exactly 0 for equal
    matrices, also for the slightly non-orthonormal float32-derived ones of look_pose"""
    return math.degrees(2 * math.asin(min(1.0, np.linalg.norm(Ra - Rb) / (2 * math.sqrt(2)))))


def pose(R, t):
    """float64 [4, 4] of [R | t] (translation_oracle.pose is the rasterizer's float32 one)"""
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def render(mesh, R, t, K=K4):
    """render_depth of one pose at H x W -> float32 [H, W] on the GPU"""
    from nope_b200.vsd import render_depth
    return render_depth(mesh, torch.from_numpy(to.pose(R, t)), K, (H, W))[0]


def inside(m):
    """the silhouette m [H, W] (torch) is not empty and touches no frame border"""
    rows, cols = m.any(1).nonzero(), m.any(0).nonzero()
    return len(rows) > 0 and rows.min() > 0 and cols.min() > 0 and rows.max() < H - 1 and cols.max() < W - 1


def perturb(rng, R, t, deg=5.0, mm=10.0):
    """(R, t) turned by deg / 2 ... deg about a random axis and moved by mm / 2 ... mm in a random direction"""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    d = rng.normal(size=3)
    return rotvec(axis * math.radians(rng.uniform(0.5, 1.0) * deg)) @ R, t + d / np.linalg.norm(d) * \
        rng.uniform(0.5, 1.0) * mm


def scene(mesh, seed, F, P, K=None, sensor=True, background=True, deg=5.0, mm=10.0):
    """F frames, a true pose each at 400 - 900 mm with the object inside the frame, and P perturbed hypotheses:
    -> (R_true [F, 3, 3], t_true [F, 3], S float64 [F, H, W] on the GPU, masks uint8 [F, H, W], R0 [F, P, 3, 3],
    t0 [F, P, 3]).  S is the render at the true pose; with `sensor` quantised to 0.1 mm after seeded noise
    (sigma 0.5 mm) with 2 % seeded holes; with `background` merged by the minimum with a plane 40 mm behind it."""
    rng = np.random.default_rng(seed)
    K = np.repeat(K4[None], F, 0) if K is None else K
    Rt, tt, S, M = [], [], [], []
    while len(Rt) < F:
        f = len(Rt)
        R = rot(rng)
        z = rng.uniform(400.0, 900.0)
        t = np.array([rng.uniform(-0.15, 0.15) * z, rng.uniform(-0.15, 0.15) * z, z])
        d = render(mesh, R, t, K[f]).double()
        m = d > 0
        if not inside(m):
            continue
        if background:
            d = torch.where(m, d, torch.full_like(d, z + 40.0))
        if sensor:
            g = torch.Generator(device=d.device).manual_seed(seed * 1000 + f)
            d = d + 0.5 * torch.randn(d.shape, generator=g, device=d.device, dtype=torch.float64)
            d = torch.round(d * 10.0) / 10.0
            d = torch.where(torch.rand(d.shape, generator=g, device=d.device) < 0.02, torch.zeros_like(d), d)
        Rt.append(R), tt.append(t), S.append(d), M.append(m.to(torch.uint8))
    R0 = np.zeros((F, P, 3, 3))
    t0 = np.zeros((F, P, 3))
    for f in range(F):
        for p in range(P):
            R0[f, p], t0[f, p] = perturb(rng, Rt[f], tt[f], deg, mm)
    return np.stack(Rt), np.stack(tt), torch.stack(S), torch.stack(M), R0, t0


def occluder():
    from nope_b200.vsd import Mesh
    return Mesh(*ro.sphere(OCC_RADIUS, 2))


def occluded_scene(mesh, seed, F, cover, behind=False, K=K4):
    """F frames: a true pose each, the target's visible mask M and the occluders O (uint8 [F, H, W] on the GPU), and
    the coverage achieved: a sphere of radius OCC_RADIUS about as large in the image as the target and at least 120 mm
    nearer the camera,
    moved from the target's box centre along a seeded direction until it hides `cover` of the target's silhouette
    (bisection, within 0.04).  With `behind`, O also holds a box 150 mm behind the target, beside it.
    -> (R_true [F, 3, 3], t_true [F, 3], M, O, coverage [F], S the target's full silhouettes, t_occ [F, 3] the
    sphere's centres)"""
    rng = np.random.default_rng(seed)
    occ = occluder()
    fx, fy, cx, cy = K
    back = None
    if behind:
        from nope_b200.vsd import Mesh
        back = Mesh(*ro.box(80.0, 60.0, 10.0))
    Rt, tt, Ms, Os, cov, Ss, To = [], [], [], [], [], [], []
    while len(Rt) < F:
        R = rot(rng)
        z = rng.uniform(400.0, 1200.0)
        t = np.array([rng.uniform(-0.15, 0.15) * z, rng.uniform(-0.15, 0.15) * z, z])
        D = render(mesh, R, t, K)
        S = D > 0
        if not inside(S):
            continue
        n, _, r0, r1, c0, c1 = to.stats(S.cpu().numpy())
        rs = math.sqrt(n / math.pi)
        zo = min(fx * OCC_RADIUS / rs, z - 120.0)                 # in front of the target's 40 mm radius
        a = rng.uniform(0, 2 * math.pi)
        u0, v0 = (c0 + c1 + 1) / 2, (r0 + r1 + 1) / 2

        def place(d):
            u, v = u0 + d * math.cos(a), v0 + d * math.sin(a)
            to_ = np.array([(u - cx) * zo / fx, (v - cy) * zo / fy, zo])
            Do = render(occ, np.eye(3), to_, K)
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
            Db = render(back, np.eye(3), tb, K)
            assert bool((~((Db > 0) & S) | (D < Db)).all())
            O = O | (Db > 0)
        Rt.append(R), tt.append(t), Ms.append(M.to(torch.uint8)), Os.append(O.to(torch.uint8)), cov.append(c)
        Ss.append(S), To.append(to_)
    return (np.stack(Rt), np.stack(tt), torch.stack(Ms), torch.stack(Os), np.array(cov), torch.stack(Ss),
            np.stack(To))


def accuracy(mesh, diameter, name, cover, n, seed=100, iters=None):
    """-> dict of per-scene errors on occluded_scene with ("O") and without ("no O") occluders: translation fit from
    initial_translation at the true rotation ("dz_px", "reproj_px"), contour fit from a start 2.5 - 5 deg and 5 - 10 mm
    off ("t_mm", "r_deg")"""
    from nope_b200.contour_refine import refine_pose_contour
    from nope_b200.translation import DEFAULT_ITERS, estimate_translation
    R_true, t_true, M, O, _, S, _ = occluded_scene(mesh, seed, n, cover)
    box = np.array([math.sqrt((s[5] - s[4] + 1) * (s[3] - s[2] + 1)) for s in (to.stats(x) for x in S.cpu().numpy())])
    rng = np.random.default_rng(seed + 1)
    st = [perturb(rng, R_true[f], t_true[f]) for f in range(n)]
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
                    "r_deg": np.array([angle(R[f], R_true[f]) for f in range(n)])}
    return out


def with_objects(model, meshes):
    """the model with meshes {id: (Mesh, diameter)} loaded as asymmetric objects"""
    from nope_b200 import bop
    for i, (mesh, d) in meshes.items():
        info = {"diameter": d, "symmetries_discrete": [], "symmetries_continuous": []}
        model.tless_cad[i] = mesh
        model.bop_models[i] = {"diameter": d, "symmetries": bop.symmetry_transformations(info), "info": info}
    return model


def tless_batch(tmp_path, B=3, models_info=True, symmetries=()):
    """a synthetic tless_obj01 test batch: a 60 x 40 x 30 box as obj_000001.ply, synthetic noisy depth PNGs at 96 x 72,
    and models_info.json (unless not `models_info`) with the box's diameter and the discrete `symmetries`
    -> (batch, the models directory, each frame's mask: the box rendered at the true pose)"""
    import cv2
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from oracle import inputs
    v, f = ro.box(60.0, 40.0, 30.0)
    ply = tmp_path / "models"
    ply.mkdir()
    with open(ply / "obj_000001.ply", "w") as fh:
        fh.write(f"ply\nformat ascii 1.0\nelement vertex {len(v)}\nproperty float x\nproperty float y\n"
                 f"property float z\nelement face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
        fh.writelines(" ".join(repr(float(x)) for x in p) + "\n" for p in v)
        fh.writelines("3 " + " ".join(str(int(i)) for i in q) + "\n" for q in f)
    if models_info:
        info = '"diameter": %r' % float(np.linalg.norm([60.0, 40.0, 30.0]))
        if symmetries:
            info += ', "symmetries_discrete": [%s]' % ", ".join(
                "[" + ", ".join(repr(float(x)) for x in m.reshape(-1)) + "]" for m in symmetries)
        (ply / "models_info.json").write_text('{"1": {%s}}' % info)
    rel = synthetic_pose_batch(42, B)[0]
    tp = torch.from_numpy(icosphere_object_rotations(0)).float()[None].expand(B, -1, -1, -1).contiguous()
    assert rel.shape[1] == tp.shape[1]
    q, r = inputs.make_images(seed=3, batch=B)
    K = torch.tensor([[150.0, 0.0, 48.2], [0.0, 151.0, 35.9], [0.0, 0.0, 1.0]], dtype=torch.float64)
    gtR, paths, masks = tp[torch.arange(B), torch.tensor([3, 17, 30])[:B]], [], []
    trans = torch.tensor([[2.0, -3.0, 300.0], [-5.0, 1.0, 280.0], [0.0, 4.0, 320.0]])[:B, :, None]
    for b in range(B):
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = gtR[b].numpy(), trans[b, :, 0].numpy()
        d = ro.render(v, f, T, K.numpy(), (72, 96))[0].numpy()
        masks.append(d > 0)
        raw = np.round(d * 10.0 + np.random.default_rng(b).normal(0, 5.0, d.shape) * (d > 0)).clip(0).astype(np.uint16)
        paths.append(str(tmp_path / f"depth_{b}.png"))
        assert cv2.imwrite(paths[-1], raw)
    return {"query": q, "reference": r, "gt_relativeR": rel[:, 0], "all_relativeR": rel, "template_poses": tp,
            "query_pose": gtR, "query_translation": trans, "intrinsic": K[None].expand(B, 3, 3).contiguous(),
            "depth_path": paths, "obj_id": torch.ones(B, dtype=torch.int64)}, str(ply), torch.from_numpy(np.stack(masks))
