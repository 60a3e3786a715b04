"""TEST INFRASTRUCTURE ONLY -- the depth rasterizer and the VSD kernel of nope_b200/csrc/render.cuh restated in torch
on the CPU, op by op in the kernels' order (DESIGN.md section 12), plus small mesh builders for the tests and
tools/vsd_time.py.

Conventions (shared with the kernel):
  * pixel (r, c) samples the image point (u, v) = (c + 1/2, r + 1/2); u = fx X / Z + cx, v = fy Y / Z + cy;
  * camera coordinates ((m0 X + m1 Y) + m2 Z) + m3 per row and the projection in float32, every product, quotient
    and sum rounded on its own;
  * fixed point: round-half-even(u * 256) with |u|, |v| <= 2^20 px, else the triangle is dropped; also dropped:
    a vertex with Z < znear, area 0, an index outside [0, V);
  * vertex order: rotated so the lowest index comes first, then oriented to positive area (no culling);
  * coverage: int64 edge functions, a sample on an edge belongs to it when the edge is top-left
    (dy < 0, or dy == 0 and dx > 0, in y-down image coordinates);
  * depth: ((w0 / Za + w1 / Zb) + w2 / Zc) in float64 with 1/Z first, area / that, rounded once to float32; the
    minimum per pixel; 0 where nothing is hit.
"""
import numpy as np
import torch

SUB = 256
MAX_COORD = float(2 ** 20)


def _project(v, pose, fx, fy, cx, cy, znear):
    m = pose.to(torch.float32)
    X, Y, Z = v[:, 0], v[:, 1], v[:, 2]

    def row(i):
        return ((m[i, 0] * X + m[i, 1] * Y) + m[i, 2] * Z) + m[i, 3]
    xc, yc, zc = row(0), row(1), row(2)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)          # noqa: E731
    u = (f32(fx) * xc) / zc + f32(cx)
    w = (f32(fy) * yc) / zc + f32(cy)
    ok = (zc >= f32(znear)) & (u.abs() <= MAX_COORD) & (w.abs() <= MAX_COORD)
    ui = torch.where(ok, torch.round(u * SUB), torch.zeros_like(u)).to(torch.int64)
    vi = torch.where(ok, torch.round(w * SUB), torch.zeros_like(w)).to(torch.int64)
    return ui, vi, zc, ok


def canonical_faces(faces):
    """rotate every face so its lowest vertex index comes first"""
    f = torch.as_tensor(faces, dtype=torch.int64)
    a = torch.where((f[:, 1] < f[:, 0]) & (f[:, 1] <= f[:, 2]), 1,
                    torch.where((f[:, 2] < f[:, 0]) & (f[:, 2] < f[:, 1]), 2, 0))
    idx = (a[:, None] + torch.arange(3)[None]) % 3
    return f.gather(1, idx)


def _top_left(dx, dy):
    return (dy < 0) | ((dy == 0) & (dx > 0))


def render(vertices, faces, poses, K, image_size, znear=0.05):
    """-> float32 [P, H, W] depth, as depth_raster_kernel computes it.  K (fx, fy, cx, cy) or [3, 3]."""
    v = torch.as_tensor(np.asarray(vertices), dtype=torch.float32)
    f = torch.as_tensor(np.asarray(faces), dtype=torch.int64)
    poses = torch.as_tensor(np.asarray(poses), dtype=torch.float32)
    if poses.dim() == 2:
        poses = poses[None]
    K = np.asarray(K, dtype=np.float64)
    fx, fy, cx, cy = (K[0, 0], K[1, 1], K[0, 2], K[1, 2]) if K.shape == (3, 3) else tuple(K)
    fx, fy, cx, cy, znear = (float(np.float32(x)) for x in (fx, fy, cx, cy, znear))
    H, W = image_size
    valid = ((f >= 0) & (f < len(v))).all(dim=1)
    f = canonical_faces(f[valid])
    out = torch.full((len(poses), H * W), float("inf"), dtype=torch.float32)
    pc = torch.arange(W, dtype=torch.int64) * SUB + SUB // 2
    pr = torch.arange(H, dtype=torch.int64) * SUB + SUB // 2
    for p in range(len(poses)):
        ui, vi, zc, ok = _project(v, poses[p], fx, fy, cx, cy, znear)
        for i0, i1, i2 in f.tolist():
            if not (ok[i0] and ok[i1] and ok[i2]):
                continue
            ax, ay, bx, by, cx_, cy_ = (int(ui[i0]), int(vi[i0]), int(ui[i1]), int(vi[i1]), int(ui[i2]), int(vi[i2]))
            za, zb, zcc = zc[i0], zc[i1], zc[i2]
            area = (bx - ax) * (cy_ - ay) - (by - ay) * (cx_ - ax)
            if area == 0:
                continue
            if area < 0:
                bx, by, cx_, cy_, zb, zcc = cx_, cy_, bx, by, zcc, zb
                area = -area
            c0 = max(0, -((128 - min(ax, bx, cx_)) >> 8)); c1 = min(W - 1, (max(ax, bx, cx_) - 128) >> 8)
            r0 = max(0, -((128 - min(ay, by, cy_)) >> 8)); r1 = min(H - 1, (max(ay, by, cy_) - 128) >> 8)
            if c0 > c1 or r0 > r1:
                continue
            px = pc[c0:c1 + 1][None, :]
            py = pr[r0:r1 + 1][:, None]
            w0 = (cx_ - bx) * (py - by) - (cy_ - by) * (px - bx)
            w1 = (ax - cx_) * (py - cy_) - (ay - cy_) * (px - cx_)
            w2 = (bx - ax) * (py - ay) - (by - ay) * (px - ax)
            inside = ((w0 > 0) | ((w0 == 0) & bool(_top_left(cx_ - bx, cy_ - by)))) & \
                     ((w1 > 0) | ((w1 == 0) & bool(_top_left(ax - cx_, ay - cy_)))) & \
                     ((w2 > 0) | ((w2 == 0) & bool(_top_left(bx - ax, by - ay))))
            if not inside.any():
                continue
            one = torch.tensor(1.0, dtype=torch.float64)
            iza, izb, izc = one / za.double(), one / zb.double(), one / zcc.double()
            s = (w0.double() * iza + w1.double() * izb) + w2.double() * izc
            d = (torch.tensor(float(area), dtype=torch.float64) / s).float()
            d = torch.where(inside, d, torch.tensor(float("inf")))
            blk = out[p].view(H, W)[r0:r1 + 1, c0:c1 + 1]
            out[p].view(H, W)[r0:r1 + 1, c0:c1 + 1] = torch.minimum(blk, d)
    out[torch.isinf(out)] = 0.0
    return out.view(len(poses), H, W)


# ------------------------------------------------------------------ VSD (vsd_kernel)
def dist_image(depth, K):
    """depth_im_to_dist_im_fast (reference src/poses/vsd_utils.py:40-62) in numpy's order: depth widened to float64"""
    depth = np.asarray(depth)
    K = np.asarray(K, dtype=np.float64)
    fx, fy, cx, cy = (K[0, 0], K[1, 1], K[0, 2], K[1, 2]) if K.shape == (3, 3) else tuple(K)
    xs, ys = np.meshgrid(np.arange(depth.shape[1]), np.arange(depth.shape[0]))
    pre_x = (xs - cx) / np.float64(fx)
    pre_y = (ys - cy) / np.float64(fy)
    return np.sqrt(np.multiply(pre_x, depth) ** 2 + np.multiply(pre_y, depth) ** 2 + depth.astype(np.float64) ** 2)


def visib_masks(dist_test, dist_gt, dist_est, delta):
    """bop19 visibility masks of the ground-truth and the estimated pose (vsd_utils.py:65-134)"""
    t32 = dist_test.astype(np.float32)
    d32 = np.float32(delta)
    gt = ((dist_gt.astype(np.float32) - t32 <= d32) | (dist_test == 0)) & (dist_gt > 0)
    est = ((dist_est.astype(np.float32) - t32 <= d32) | (dist_test == 0)) & (dist_est > 0)
    return gt, est | (gt & (dist_est > 0))


def vsd(depth_test, depth_gt, depth_est, K, delta=15, tau=20, cost_type="step"):
    """float64 [P] for one frame: depth_test [H, W] float64, depth_gt [H, W], depth_est [P, H, W] float32"""
    dt = dist_image(depth_test, K)
    dg = dist_image(depth_gt, K)
    out = np.zeros(len(depth_est))
    for p in range(len(depth_est)):
        de = dist_image(depth_est[p], K)
        gt, est = visib_masks(dt, dg, de, delta)
        inter, union = gt & est, gt | est
        nu, ni = int(union.sum()), int(inter.sum())
        if nu == 0:
            out[p] = 1.0
            continue
        dd = np.abs(dg[inter] - de[inter])
        if cost_type == "step":
            out[p] = (int(np.sum(dd >= tau)) + (nu - ni)) / float(nu)      # integers: exact until the division
        else:
            out[p] = (float(np.sum(np.minimum(dd / tau, 1.0))) + (nu - ni)) / float(nu)
    return out


# ------------------------------------------------------------------ meshes
def box(sx=60.0, sy=40.0, sz=30.0):
    """closed box centred at the origin, 8 vertices, 12 triangles, outward winding"""
    v = np.array([[x, y, z] for x in (-sx / 2, sx / 2) for y in (-sy / 2, sy / 2) for z in (-sz / 2, sz / 2)],
                 dtype=np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                  [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    return v, f


def sphere(radius=40.0, subdivisions=2):
    """icosphere: 20 * 4^subdivisions triangles"""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdivisions):
        mid, nf = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[key] = len(v) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.array(v) * radius).astype(np.float32), np.array(f, dtype=np.int32)


def plane(nx=8, ny=6, sx=80.0, sy=60.0):
    """tessellated plane z = 0 over [-sx/2, sx/2] x [-sy/2, sy/2], 2 nx ny triangles"""
    xs, ys = np.linspace(-sx / 2, sx / 2, nx + 1), np.linspace(-sy / 2, sy / 2, ny + 1)
    v = np.array([[x, y, 0.0] for y in ys for x in xs], dtype=np.float32)
    f = []
    for j in range(ny):
        for i in range(nx):
            a = j * (nx + 1) + i
            f += [[a, a + 1, a + nx + 2], [a, a + nx + 2, a + nx + 1]]
    return v, np.array(f, dtype=np.int32)


def soup(n=64, seed=0, extent=50.0, size=15.0):
    """n random triangles in a cube, unconnected"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-extent / 2, extent / 2, size=(n, 1, 3))
    v = (c + rng.uniform(-size, size, size=(n, 3, 3))).reshape(-1, 3).astype(np.float32)
    return v, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def look_pose(rx=0.0, ry=0.0, rz=0.0, t=(0.0, 0.0, 400.0)):
    """float32 [4, 4] model -> camera: R = Rz Ry Rx (radians), translation t (mm)"""
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T.astype(np.float32)
