"""T-LESS evaluation on the GPU (DESIGN.md section 12): PLY meshes, a depth rasterizer standing in for pyrender's
DEPTH_ONLY render (reference src/poses/vsd.py:25-55) and the VSD error of `vsd_obj` (src/poses/vsd.py:92-135,
src/poses/vsd_utils.py, visibility mode "bop19").  Both hot paths are CUDA kernels (render.cuh); there is no CPU
fallback."""

import numpy as np
import torch

from . import _lib

COST_TYPES = {"step": 0, "tlinear": 1}          # NOPE_VSD_* of include/nope_b200.h
MAX_SIDE = 8192
MAX_TAUS = 16                                   # tolerances of one multi-tau VSD pass
_stream = _lib.stream                           # the name the render and pose-fit tests import

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _parse_header(f):
    if f.readline().strip() != b"ply":
        raise ValueError("not a PLY file")
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise ValueError("PLY header has no end_header")
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if not elements:
                raise ValueError("PLY property before any element")
            if tok[1] == "list":
                elements[-1][2].append((tok[4], "list", tok[2], tok[3]))
            else:
                elements[-1][2].append((tok[2], tok[1], None, None))
        elif tok[0] == "end_header":
            break
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError(f"PLY format {fmt!r} is not supported (ascii, binary_little_endian)")
    for _, _, props in elements:
        for _, typ, cnt, item in props:
            for t in ((cnt, item) if typ == "list" else (typ,)):
                if t not in _PLY_TYPES:
                    raise ValueError(f"PLY property type {t!r} is not supported")
    return fmt, elements


def _triangle_rows(body, pos, count, props):
    """Binary element rows read in one structured read, assuming every list property holds 3 entries (the triangle
    meshes of BOP / T-LESS): -> (columns, new offset), or None when that assumption does not hold, and the caller
    parses row by row."""
    fields = []
    for pname, typ, cnt, item in props:
        if typ == "list":
            fields += [(pname + "#n", "<" + _PLY_TYPES[cnt]), (pname, "<" + _PLY_TYPES[item], (3,))]
        else:
            fields.append((pname, "<" + _PLY_TYPES[typ]))
    dt = np.dtype(fields)
    if pos + count * dt.itemsize > len(body):
        return None
    arr = np.frombuffer(body, dtype=dt, count=count, offset=pos)
    if any(typ == "list" and not (arr[pname + "#n"] == 3).all() for pname, typ, _, _ in props):
        return None
    return {p[0]: arr[p[0]].astype(np.int64) if p[1] == "list" else arr[p[0]] for p in props}, \
        pos + count * dt.itemsize


def _faces_from_rows(rows, name):
    if isinstance(rows, np.ndarray):                  # the structured read: 3 entries per row by construction
        return rows
    if any(len(r) != 3 for r in rows):
        raise ValueError(f"PLY face list {name!r} holds a face that is not a triangle")
    return rows


def read_ply(path):
    """-> (vertices float32 [V, 3], faces int32 [F, 3]) of an ascii or binary_little_endian PLY file: float or double
    x y z (other vertex properties are skipped), faces from a `vertex_indices` / `vertex_index` list of any integer
    types.  A face that is not a triangle or an index outside [0, V) raises ValueError."""
    with open(path, "rb") as f:
        fmt, elements = _parse_header(f)
        body = f.read()
    data, pos = {}, 0
    tokens = body.decode("ascii").split() if fmt == "ascii" else None
    for name, count, props in elements:
        if fmt == "ascii":
            cols = {p[0]: [] for p in props}
            for _ in range(count):
                for pname, typ, cnt, item in props:
                    if typ == "list":
                        n = int(tokens[pos])
                        cols[pname].append([int(float(t)) for t in tokens[pos + 1:pos + 1 + n]])
                        pos += 1 + n
                    else:
                        cols[pname].append(float(tokens[pos]))
                        pos += 1
        elif all(p[1] != "list" for p in props):                    # fixed-size rows: one structured read
            dt = np.dtype([(p[0], "<" + _PLY_TYPES[p[1]]) for p in props])
            arr = np.frombuffer(body, dtype=dt, count=count, offset=pos)
            pos += count * dt.itemsize
            cols = {p[0]: arr[p[0]] for p in props}
        elif (fast := _triangle_rows(body, pos, count, props)) is not None:   # every list holds 3 entries
            cols, pos = fast
        else:
            cols = {p[0]: [] for p in props}
            for _ in range(count):
                for pname, typ, cnt, item in props:
                    if typ == "list":
                        cdt = np.dtype("<" + _PLY_TYPES[cnt])
                        n = int(np.frombuffer(body, dtype=cdt, count=1, offset=pos)[0])
                        pos += cdt.itemsize
                        idt = np.dtype("<" + _PLY_TYPES[item])
                        cols[pname].append(np.frombuffer(body, dtype=idt, count=n, offset=pos).astype(np.int64).tolist())
                        pos += n * idt.itemsize
                    else:
                        vdt = np.dtype("<" + _PLY_TYPES[typ])
                        cols[pname].append(np.frombuffer(body, dtype=vdt, count=1, offset=pos)[0])
                        pos += vdt.itemsize
        data[name] = cols
    if "vertex" not in data or not all(k in data["vertex"] for k in "xyz"):
        raise ValueError("PLY file has no vertex element with x, y, z")
    vx = data["vertex"]
    vertices = np.stack([np.asarray(vx[k], dtype=np.float64) for k in "xyz"], axis=1).astype(np.float32)
    face = data.get("face", {})
    key = next((k for k in ("vertex_indices", "vertex_index") if k in face), None)
    if key is None:
        raise ValueError("PLY file has no face element with vertex_indices / vertex_index")
    rows = _faces_from_rows(face[key], key)
    faces = np.asarray(rows, dtype=np.int64).reshape(-1, 3)
    if faces.size and (faces.min() < 0 or faces.max() >= len(vertices)):
        raise ValueError(f"PLY face index outside [0, {len(vertices)})")
    return vertices, faces.astype(np.int32)


class Mesh:
    """Device copy of a triangle mesh: vertices float32 [V, 3] (mm, model frame), faces int32 [F, 3].  The face indices
    are checked once, here, on the host."""

    def __init__(self, vertices, faces, device="cuda"):
        v = torch.as_tensor(np.asarray(vertices) if not torch.is_tensor(vertices) else vertices)
        fc = torch.as_tensor(np.asarray(faces) if not torch.is_tensor(faces) else faces)
        if v.dim() != 2 or v.shape[1] != 3 or v.shape[0] < 1:
            raise ValueError(f"vertices [V, 3] with V >= 1 expected, got {tuple(v.shape)}")
        if fc.dim() != 2 or fc.shape[1] != 3 or fc.shape[0] < 1:
            raise ValueError(f"faces [F, 3] with F >= 1 expected, got {tuple(fc.shape)}")
        if fc.is_floating_point() or fc.dtype == torch.bool:
            raise ValueError(f"faces must be integers, got {fc.dtype}")
        fc64 = fc.cpu().to(torch.int64)
        if int(fc64.min()) < 0 or int(fc64.max()) >= v.shape[0]:
            raise ValueError(f"face index outside [0, {v.shape[0]})")
        self.vertices = v.to(device=device, dtype=torch.float32).contiguous()
        self.faces = fc64.to(torch.int32).to(device).contiguous()
        v64 = v.detach().cpu().to(torch.float32).to(torch.float64)
        self.radius = float(torch.sqrt((v64 * v64).sum(1)).max())    # the largest vertex norm (mm)

    @classmethod
    def from_ply(cls, path, device="cuda"):
        return cls(*read_ply(path), device=device)

    @property
    def device(self):
        return self.vertices.device

    @property
    def num_faces(self):
        return self.faces.shape[0]


def _intrinsics(K):
    K = torch.as_tensor(np.asarray(K) if not torch.is_tensor(K) else K).detach().cpu().to(torch.float64)
    if K.shape == (3, 3):
        return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    if K.shape == (4,):
        return tuple(float(x) for x in K)
    raise ValueError(f"K [3, 3] or (fx, fy, cx, cy) expected, got {tuple(K.shape)}")


def _image_size(image_size):
    if len(image_size) != 2:
        raise ValueError(f"image_size (H, W) expected, got {image_size!r}")
    H, W = int(image_size[0]), int(image_size[1])
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
        raise ValueError(f"H and W must be in [1, {MAX_SIDE}], got {(H, W)}")
    return H, W



def render_depth(mesh, poses, K, image_size, znear=0.05):
    """Camera-Z depth (float32 [P, H, W], 0 where nothing is hit) of `mesh` under poses [P, 4, 4] or [4, 4]
    (model -> OpenCV camera, mm), intrinsics K [3, 3] or (fx, fy, cx, cy), image_size (H, W).  znear 0.05 is the
    reference's (src/poses/vsd.py:43).  Pixel (r, c) samples the image point (c + 1/2, r + 1/2); the intrinsics and
    the poses are rounded to float32.  Runs on mesh's device, on the current stream, without synchronising."""
    if not isinstance(mesh, Mesh):
        raise ValueError("mesh must be a nope_b200.vsd.Mesh")
    dev = mesh.device
    if dev.type != "cuda":
        raise _lib.NopeError("render_depth needs a CUDA mesh (no CPU fallback)")
    poses = torch.as_tensor(poses) if not torch.is_tensor(poses) else poses
    if poses.dim() == 2:
        poses = poses[None]
    if poses.dim() != 3 or poses.shape[1:] != (4, 4) or poses.shape[0] < 1:
        raise ValueError(f"poses [P, 4, 4] expected, got {tuple(poses.shape)}")
    fx, fy, cx, cy = _intrinsics(K)
    H, W = _image_size(image_size)
    if not znear > 0:
        raise ValueError(f"znear must be > 0, got {znear}")
    p = poses.to(device=dev, dtype=torch.float32).contiguous()
    out = torch.empty((p.shape[0], H, W), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_render_depth(
            _lib.ptr(mesh.vertices), mesh.vertices.shape[0], _lib.ptr(mesh.faces), mesh.num_faces, _lib.ptr(p),
            p.shape[0], fx, fy, cx, cy, float(znear), H, W, _lib.ptr(out), _lib.stream(dev)))
    return out


def vsd_errors(depth_test, depth_gt, depth_est, K, delta=15, tau=20, cost_type="step"):
    """VSD errors float64 [F, P] of P estimated poses per frame, as `vsd_obj` (src/poses/vsd.py:92-135) computes them:
      depth_test [F, H, W] (the sensor depth in mm, the PNG / 10.0; widened to float64),
      depth_gt   [F, H, W] float32 (the model rendered at the ground-truth pose),
      depth_est  [F, P, H, W] float32 (the model rendered at the estimated poses),
      K          [F, 3, 3] or [F, 4] (fx, fy, cx, cy), float64.
    delta, tau and cost_type default to vsd_obj's.  The three depth tensors must be on one CUDA device.
    A 1-D `tau` of T <= 16 tolerances scores all of them in one pass and returns [F, P, T]; entry [..., j] equals the
    scalar call at tau[j] bit for bit.  K is then read on the host (DESIGN.md section 15)."""
    if cost_type not in COST_TYPES:
        raise ValueError(f"unknown cost_type {cost_type!r} (supported: {sorted(COST_TYPES)})")
    if not float(delta) >= 0:
        raise ValueError(f"delta must be >= 0, got {delta}")
    if np.ndim(tau) == 1:
        return _vsd_errors_taus(depth_test, depth_gt, depth_est, K, delta, tau, cost_type)
    if not float(tau) > 0:
        raise ValueError(f"tau must be > 0, got {tau}")
    if depth_test.dim() != 3 or depth_gt.shape != depth_test.shape or depth_est.dim() != 4 or \
            depth_est.shape[0] != depth_test.shape[0] or depth_est.shape[2:] != depth_test.shape[1:]:
        raise ValueError(f"depth_test [F, H, W], depth_gt [F, H, W] and depth_est [F, P, H, W] expected, got "
                         f"{tuple(depth_test.shape)}, {tuple(depth_gt.shape)}, {tuple(depth_est.shape)}")
    F_, P, H, W = depth_est.shape
    if F_ < 1 or P < 1:
        raise ValueError("empty batch")
    _image_size((H, W))
    dev = depth_est.device
    if dev.type != "cuda" or depth_gt.device != dev or depth_test.device != dev:
        raise _lib.NopeError("vsd_errors needs the three depth tensors on one CUDA device (no CPU fallback)")
    K = torch.as_tensor(np.asarray(K) if not torch.is_tensor(K) else K)
    if K.dim() == 3 and K.shape[1:] == (3, 3):
        K = torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], dim=1)
    if K.shape != (F_, 4):
        raise ValueError(f"K [F, 3, 3] or [F, 4] with F = {F_} expected, got {tuple(K.shape)}")
    k = K.to(device=dev, dtype=torch.float64).contiguous()
    dt = depth_test.to(torch.float64).contiguous()
    dg = depth_gt.to(torch.float32).contiguous()
    de = depth_est.to(torch.float32).contiguous()
    out = torch.empty((F_, P), device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_vsd_error(
            _lib.ptr(dt), _lib.ptr(dg), _lib.ptr(de), F_, P, H, W, _lib.ptr(k), float(delta), float(tau),
            COST_TYPES[cost_type], _lib.ptr(out), _lib.stream(dev)))
    return out


def _vsd_errors_taus(depth_test, depth_gt, depth_est, K, delta, tau, cost_type):
    taus = np.asarray(tau.detach().cpu() if torch.is_tensor(tau) else tau, dtype=np.float64)
    if not 1 <= len(taus) <= MAX_TAUS:
        raise ValueError(f"1 to {MAX_TAUS} tolerances expected, got {len(taus)}")
    if not (np.isfinite(taus).all() and (taus > 0).all()):
        raise ValueError(f"every tau must be finite and > 0, got {taus.tolist()}")
    if depth_test.dim() != 3 or depth_gt.shape != depth_test.shape or depth_est.dim() != 4 or \
            depth_est.shape[0] != depth_test.shape[0] or depth_est.shape[2:] != depth_test.shape[1:]:
        raise ValueError(f"depth_test [F, H, W], depth_gt [F, H, W] and depth_est [F, P, H, W] expected, got "
                         f"{tuple(depth_test.shape)}, {tuple(depth_gt.shape)}, {tuple(depth_est.shape)}")
    F_, P, H, W = depth_est.shape
    if F_ < 1 or P < 1:
        raise ValueError("empty batch")
    _image_size((H, W))
    dev = depth_est.device
    if dev.type != "cuda" or depth_gt.device != dev or depth_test.device != dev:
        raise _lib.NopeError("vsd_errors needs the three depth tensors on one CUDA device (no CPU fallback)")
    K = torch.as_tensor(np.asarray(K) if not torch.is_tensor(K) else K).detach().cpu().to(torch.float64)
    if K.dim() == 3 and K.shape[1:] == (3, 3):
        K = torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], dim=1)
    if K.shape != (F_, 4):
        raise ValueError(f"K [F, 3, 3] or [F, 4] with F = {F_} expected, got {tuple(K.shape)}")
    k = K.contiguous()
    if not torch.isfinite(k).all() or (k[:, :2] == 0).any():
        raise ValueError("intrinsics must be finite with fx and fy non-zero")
    taus = np.ascontiguousarray(taus)
    dt = depth_test.to(torch.float64).contiguous()
    dg = depth_gt.to(torch.float32).contiguous()
    de = depth_est.to(torch.float32).contiguous()
    out = torch.empty((F_, P, len(taus)), device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_vsd_error_taus(
            _lib.ptr(dt), _lib.ptr(dg), _lib.ptr(de), F_, P, H, W, k.data_ptr(), float(delta), COST_TYPES[cost_type],
            taus.ctypes.data, len(taus), _lib.ptr(out), _lib.stream(dev)))
    return out
