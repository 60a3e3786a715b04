"""Pose-grid host utilities (reference: src/poses/utils.py:72-102,
src/poses/rotation_conversions.py:490-503, src/dataloader/shapeNet.py:243-250,302-307)."""
import numpy as np
import torch


def matrix_to_rotation_6d(matrix):
    """First two rows of R, flattened (rotation_conversions.py:490-503)."""
    return matrix[..., :2, :].clone().reshape(*matrix.shape[:-2], 6)


def relative_rotation_6d(template_R, ref_R):
    """all_relativeR[n] = rot6d(R_template[n] @ inv(R_ref))  (shapeNet.py:243-250, 302-307).
    template_R [N,3,3], ref_R [3,3] (numpy float64) -> torch float32 [N,6]."""
    rel = np.asarray(template_R) @ np.linalg.inv(np.asarray(ref_R))
    return matrix_to_rotation_6d(torch.tensor(rel, dtype=torch.float32))


def _icosphere(level):
    """Vertices of an icosahedron subdivided `level + 1` times: 42 / 162 / 642 / 2562 /
    10242 points for level 0..4, the sizes of the reference's shipped grids (SURVEY.md F10).
    The reference's .npy grids come from Blender's icosphere; vertex ORDER differs, the
    point set is the same construction."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t),
         (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    verts = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4),
             (11, 10, 2), (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8),
             (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(level + 1):
        cache = {}

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                cache[key] = len(verts) - 1
            return cache[key]
        nf = []
        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    return np.stack(verts)


def icosphere_object_rotations(level, upper_only=False):
    """Synthetic pose grid: object rotations whose camera sits at each icosphere vertex
    looking at the origin.  [N,3,3] float64."""
    pts = _icosphere(level)
    if upper_only:
        pts = pts[pts[:, 2] >= 0]
    return viewpoint_rotations(pts)


def viewpoint_rotations(pts):
    """Object rotations whose camera sits at each point pts [N, 3] looking at the origin, built as the icosphere
    grids are (the same up-vector rule).  [N,3,3] float64."""
    Rs = []
    for p in pts:
        z = p / np.linalg.norm(p)
        up = np.array([0.0, 0.0, 1.0]) if abs(z[2]) < 0.999 else np.array([0.0, 1.0, 0.0])
        x = np.cross(up, z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        Rs.append(np.stack([x, y, z]))      # world -> camera
    return np.stack(Rs)


def inplane_expand(R, n_inplane):
    """Every grid rotation combined with `n_inplane` in-plane rotations (about the camera's optical
    axis, z): [N,3,3] -> [N * n_inplane, 3,3], in-plane index fastest.  BASELINE configs[3]'s "10k
    hypotheses" = the level-3 grid (2562 viewpoints) x 4 in-plane rotations = 10248 (SURVEY.md 8d)."""
    out = []
    for a in range(n_inplane):
        t = 2.0 * np.pi * a / n_inplane
        Rz = np.array([[np.cos(t), -np.sin(t), 0.0], [np.sin(t), np.cos(t), 0.0], [0.0, 0.0, 1.0]])
        out.append(Rz[None] @ R)
    return np.stack(out, axis=1).reshape(-1, 3, 3)


def synthetic_pose_batch(n_poses, batch, seed=0):
    """[B,N,6] relative rotations for benchmarking: icosphere grids for the sizes the
    reference ships (42/162/642/2562/10242), the level-3 grid x 4 in-plane rotations for 10248,
    seeded random rotations otherwise."""
    sizes = {42: 0, 162: 1, 642: 2, 2562: 3, 10242: 4}
    g = torch.Generator().manual_seed(seed)
    if n_poses in sizes:
        R = icosphere_object_rotations(sizes[n_poses])
    elif n_poses == 10248:
        R = inplane_expand(icosphere_object_rotations(3), 4)
    else:
        q = torch.randn((n_poses, 4), generator=g, dtype=torch.float64)
        q = q / q.norm(dim=1, keepdim=True)
        w, x, y, z = q.unbind(1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
                        dim=1).reshape(n_poses, 3, 3).numpy()
    out = []
    for b in range(batch):
        ref = R[(7 + 3 * b) % len(R)]
        out.append(relative_rotation_6d(R, ref))
    return torch.stack(out), torch.from_numpy(np.ascontiguousarray(R))
