"""Plain-torch restatement of the in-plane rotation search (nope_b200/inplane.py and inplane_rotate_kernel): the
rotated crops op by op in float32, one rounding per product and per sum in the kernel's order (the oracle the GPU
tests hold the kernel to bit for bit), a float64 pinhole projection for the geometry of the convention, and the
joint top-k over (angle, pose)."""
import torch


def rotate(images, cossin):
    """images [B, 3, H, W], cossin [A, 2] float32 -> [B, A, 3, H, W]: I_a(x, y) = I(c + R2(alpha_a) ((x, y) - c)),
    bilinear, taps outside the image -1.  Order: source coordinates, floor, fractions, the two row lerps, the
    column lerp."""
    img, cs = images.cpu().float(), cossin.cpu().float()
    B, _, H, W = img.shape
    A = cs.shape[0]
    c, s = cs[:, 0].view(A, 1, 1), cs[:, 1].view(A, 1, 1)
    cx = torch.tensor(float(W - 1), dtype=torch.float32) * 0.5
    cy = torch.tensor(float(H - 1), dtype=torch.float32) * 0.5
    dx = torch.arange(W, dtype=torch.float32).view(1, 1, W) - cx
    dy = torch.arange(H, dtype=torch.float32).view(1, H, 1) - cy
    sx = (c * dx - s * dy) + cx                                                    # [A, H, W]
    sy = (s * dx + c * dy) + cy
    x0, y0 = torch.floor(sx), torch.floor(sy)
    fx, fy = sx - x0, sy - y0
    ix, iy = x0.long(), y0.long()

    def tap(yy, xx):
        inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = img[:, :, yy.clamp(0, H - 1), xx.clamp(0, W - 1)]                      # [B, 3, A, H, W]
        return torch.where(inside, v, torch.tensor(-1.0)).permute(0, 2, 1, 3, 4)

    v00, v01, v10, v11 = tap(iy, ix), tap(iy, ix + 1), tap(iy + 1, ix), tap(iy + 1, ix + 1)
    fx, fy = fx[None, :, None], fy[None, :, None]
    top = v00 + fx * (v01 - v00)
    bot = v10 + fx * (v11 - v10)
    return (top + fy * (bot - top)).contiguous()


def project(R, t, X, f, c):
    """float64 pinhole: points X [n, 3] under the pose (R [3, 3], t [3]) -> pixels [n, 2] = f (RX + t)_xy / z + c"""
    Y = X.double() @ R.double().T + t.double()
    return f * Y[:, :2] / Y[:, 2:3] + torch.as_tensor(c, dtype=torch.float64)


def joint_topk(sim, k):
    """sim [..., A, N] -> (nearest_idx, angle_idx) [..., k]: descending over the flat a * N + n, ties -> lowest"""
    A, N = sim.shape[-2:]
    flat = sim.cpu().reshape(-1, A * N)
    order = torch.sort(-flat, dim=1, stable=True).indices[:, :k].reshape(sim.shape[:-2] + (k,))
    return order % N, order // N
