"""In-plane rotation search (DESIGN.md section 11): the convention, in one place.

The template grids have no roll about the viewing axis, while a query crop keeps whatever roll its camera had.
The search rotates each query crop by A angles and scores every rotated copy against the same templates:
  * angles alpha_a = a * 360 / A degrees, a = 0 .. A-1, 1 <= A <= 360 (an integer A, no explicit angle lists);
  * rotated copy a: I_a(x, y) = I(c + R2(alpha_a) ((x, y) - c)) in pixel-index coordinates (x right, y down),
    c = ((W - 1) / 2, (H - 1) / 2), R2(alpha) = [[cos, -sin], [sin, cos]], bilinear, taps outside read -1.0;
  * a match of copy a with template n means the query pose R = Rz(alpha_a) template_poses[n], Rz(alpha) =
    [[cos, -sin, 0], [sin, cos, 0], [0, 0, 1]] in the OpenCV camera frame.  In the reference's terms that is
    adding_inplane_to_pose(template, inplane=-alpha) (src/poses/utils.py:300-303), and compute_inplane(R, template)
    returns -alpha.  With square pixels and the principal point at c, projecting Rz(alpha) X moves the image point
    by R2(alpha) about c, which is why the rule holds.
cos / sin are computed on the host in float64 and rounded once to float32; quarter turns (4a a multiple of A) are
exactly 0 and +-1, so bin 0 copies the image bit for bit and the 90-degree bin of a square image equals
torch.rot90(I, 1, dims=(-2, -1))."""
import math
import numbers

import torch

from . import _lib
from ._lib import MAX_TOPK

MAX_ANGLES = 360


def check_angles(A):
    if isinstance(A, bool) or not isinstance(A, numbers.Integral) or not 1 <= A <= MAX_ANGLES:
        raise ValueError(f"angles must be an integer in [1, {MAX_ANGLES}], got {A!r}")
    return int(A)


def check_inplane_args(A, k, N):
    """A angles, top-k over A * N (angle, pose) pairs: ValueError unless 1 <= A <= 360, 1 <= k <= 64, k <= A * N."""
    A = check_angles(A)
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= MAX_TOPK:
        raise ValueError(f"k must be an integer in [1, {MAX_TOPK}], got {k!r}")
    if N < 1 or k > A * N:
        raise ValueError(f"k = {k} exceeds the {A} x {N} (angle, pose) pairs")
    return A, int(k)


def _cos_sin(A):
    """[(cos, sin)] of a * 2 pi / A in float64, quarter turns exact"""
    A = check_angles(A)
    out = []
    for a in range(A):
        if (4 * a) % A == 0:
            out.append(((1.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))[(4 * a) // A])
        else:
            t = 2.0 * math.pi * a / A
            out.append((math.cos(t), math.sin(t)))
    return out


def inplane_angles(A):
    """[A] float64 degrees, a * 360 / A"""
    A = check_angles(A)
    return torch.arange(A, dtype=torch.float64) * 360.0 / A


def inplane_table(A):
    """[A, 2] float32 (cos, sin), computed in float64 and rounded once"""
    return torch.tensor(_cos_sin(A), dtype=torch.float64).float()


def inplane_rotations(A):
    """[A, 3, 3] float64 Rz(alpha_a)"""
    cs = torch.tensor(_cos_sin(A), dtype=torch.float64)
    R = torch.zeros((len(cs), 3, 3), dtype=torch.float64)
    R[:, 0, 0], R[:, 0, 1], R[:, 1, 0], R[:, 1, 1], R[:, 2, 2] = cs[:, 0], -cs[:, 1], cs[:, 1], cs[:, 0], 1.0
    return R


_device_tables = {}


def _on_device(fn, A, device):
    """fn(A) uploaded once per device (a cached constant: later calls make no host-to-device copy)"""
    key = (fn.__name__, A, str(device))
    t = _device_tables.get(key)
    if t is None:
        t = _device_tables[key] = fn(A).to(device)
    return t


def rotate_images(images, A):
    """images [B, 3, H, W] (CUDA) -> [B, A, 3, H, W] float32: every rotated copy, materialised
    (inplane_rotate_kernel).  The search itself never forms this batch (FeatureExtractor.encode_image_inplane)."""
    A = check_angles(A)
    if images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"images [B, 3, H, W] expected, got {tuple(images.shape)}")
    if images.device.type != "cuda":
        raise _lib.NopeError("rotate_images needs CUDA tensors (no CPU fallback)")
    x = images.to(torch.float32).contiguous()
    B, _, H, W = x.shape
    out = torch.empty((B, A, 3, H, W), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().nope_inplane_rotate(
            _lib.ptr(x), B, H, W, _lib.ptr(_on_device(inplane_table, A, x.device)), A, _lib.ptr(out),
            _lib.stream(x.device)))
    return out


def compose(template_poses, pose_idx, angle_idx, A):
    """R = Rz(alpha[angle_idx]) template_poses[pose_idx] in float64, on pose_idx's device: the query pose of a
    match between rotated copy angle_idx and template pose_idx.  template_poses [N, 3, 3] (or [1, N, 3, 3])."""
    tp = template_poses[0] if template_poses.dim() == 4 else template_poses
    dev = pose_idx.device
    Rz = _on_device(inplane_rotations, check_angles(A), dev)
    return Rz[angle_idx] @ tp.to(dev, torch.float64)[pose_idx]
