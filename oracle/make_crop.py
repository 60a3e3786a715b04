"""TEST INFRASTRUCTURE ONLY -- write tests/golden/crop.npz from the UNMODIFIED reference's `crop_frame`
(src/poses/utils.py:204-272) and the input pipeline of its dataloaders: PIL's `paste` onto black through the mask
(bop.py:223-225, shapeNet.py:206-208), `crop_frame`, then the `img_transform` composition ToTensor / Resize(S) /
x*2-1 (bop.py:111-117).  The `M` crop_frame gets from cv2.getPerspectiveTransform is recorded on the way.

Cases (frames are seeded and stored once each under frame_<name>; their rows repeat, so the file stays small):
  bop_upright / bop_inplane   720x540 RGB, Primesense intrinsics, binary mask, the two keep_inplane modes, metres
  shapenet_rgba               512x512 RGBA with graded alpha, K = 525 / 256, bbox 1 (shapeNet.py:167-182)
  shapenet_axis               the same with the object on the optical axis and no rotation: crop_frame's fallback
                              of `upper` and `right` to the image axes
  odd_frame                   a 251x333 frame, graded mask, S = 17
  partly_outside / outside    a crop across the frame's border and one entirely beside it
  block_assoc                 a crop whose pixel (100, 99) tells OpenCV's 64-column coordinate blocks from the naive
                              association (its row ramp makes the 1/32 px step visible)
Stored per case (keys `<case>__<field>`): frame (the name of a stored frame), mask (empty when none), K, pose, vbs, S, keep_inplane, M (float64,
as crop_frame computes it), inv (cv2.invert of M, DECOMP_LU) and crop (uint8 [S, S, 3], the reference's output).

Run in the build container (CPU):   python -m oracle.make_crop
"""
import json
import os
import sys

import numpy as np

from . import inputs
from .crop_oracle import PRIMESENSE_K, SHAPENET_K
from .ref_import import REFERENCE_ROOT, _install_stubs


def _frame(H, W, C, seed):
    """texture as seeded random tables of x + 3 y (every row is the row above shifted by 3 px, which deflate stores
    in a few bytes), a few hard-edged rectangles, and for C = 4 an alpha graded from 0 to 255 in bands"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    d = x + 3 * y
    f = rng.integers(0, 256, (256, 3), dtype=np.uint8)[d % 256]
    for _ in range(6):
        y0, x0 = rng.integers(0, H), rng.integers(0, W)
        f[y0:y0 + rng.integers(5, H // 3 + 6), x0:x0 + rng.integers(5, W // 3 + 6)] = rng.integers(0, 256, 3)
    if C == 4:
        alpha = np.abs((d % 512) - 256).clip(0, 255).astype(np.uint8)     # a triangle wave: 0 ... 255 ... 0
        f = np.concatenate([f, alpha[..., None]], -1)
    return f


def _pose(rot_seed, t):
    from .crop_oracle import _rotation
    p = np.eye(4)
    p[:3, :3] = np.eye(3) if rot_seed is None else _rotation(np.random.default_rng(rot_seed))
    p[:3, 3] = t
    return p


def cases():
    H, W = 540, 720
    bop = _frame(H, W, 3, 1)
    yy, xx = np.mgrid[0:H, 0:W]
    bop_mask = (np.hypot(xx - 380, yy - 250) < 110).astype(np.uint8) * 255
    bop_pose = _pose(11, [0.021, -0.015, 0.653])                     # mm / 1000, as bop.py:196-199 converts
    vbs = 1.2 * 108.69 / 1000.0                                       # 1.2 * diameter (mm) / 1000
    rgba = _frame(512, 512, 4, 2)
    odd = _frame(251, 333, 3, 3)
    odd_mask = np.clip((np.mgrid[0:251, 0:333][1] - 80) * 2, 0, 255).astype(np.uint8)
    odd_K = np.array([[300.0, 0.0, 166.4], [0.0, 310.0, 125.1], [0.0, 0.0, 1.0]])
    ramp = np.repeat(((np.arange(H) * 37) % 256).astype(np.uint8)[:, None, None], W, 1).repeat(3, 2)
    sep_pose = np.array([[0.9418327109232576, 0.27957662208022427, -0.18651556777159142, 0.1970104305158223],
                         [0.17490170924830953, 0.06616203706859464, 0.9823604109251115, -0.02318938948819463],
                         [0.2869852552605577, -0.9578410605299533, 0.013415141664819663, 1.4382899181255384],
                         [0.0, 0.0, 0.0, 1.0]])
    frames = dict(bop=bop, rgba=rgba, odd=odd, ramp=ramp)
    return frames, [
        ("bop_upright", "bop", bop_mask, PRIMESENSE_K, bop_pose, vbs, 128, False),
        ("bop_inplane", "bop", bop_mask, PRIMESENSE_K, bop_pose, vbs, 128, True),
        ("shapenet_rgba", "rgba", None, SHAPENET_K, _pose(12, [0.04, -0.03, 1.35]), 1.0, 128, False),
        ("shapenet_axis", "rgba", None, SHAPENET_K, _pose(None, [0.0, 0.0, 1.2]), 1.0, 64, False),
        ("odd_frame", "odd", odd_mask, odd_K, _pose(13, [0.01, 0.02, 0.5]), 0.2, 17, False),
        ("partly_outside", "bop", None, PRIMESENSE_K, _pose(14, [0.23, 0.05, 0.7]), 0.15, 64, False),
        ("outside", "bop", None, PRIMESENSE_K, _pose(15, [0.9, 0.05, 0.7]), 0.15, 64, True),
        ("block_assoc", "ramp", None, PRIMESENSE_K, sep_pose, 0.13333522506025397, 256, True),
    ]


def write_crop(out_dir=inputs.GOLDEN_DIR):
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import cv2
    import torchvision
    from einops import rearrange
    from PIL import Image
    from torchvision import transforms
    from src.poses import utils as ref_utils

    recorded = []
    get_perspective = cv2.getPerspectiveTransform

    def record(src, dst):
        M = get_perspective(src, dst)
        recorded.append(M.copy())
        return M

    ref_utils.cv2.getPerspectiveTransform = record
    try:
        data, summary = {}, {}
        frames, all_cases = cases()
        for fname, frame in frames.items():
            data[f"frame_{fname}"] = frame
        for name, fname, mask, K, pose, vbs, S, keep_inplane in all_cases:
            frame = frames[fname]
            img_transform = transforms.Compose([
                transforms.ToTensor(), torchvision.transforms.Resize(S),
                transforms.Lambda(lambda x: rearrange(x * 2.0 - 1.0, "c h w -> h w c"))])
            src = Image.fromarray(frame)
            black = Image.new("RGB", src.size, (0, 0, 0))
            black.paste(src, mask=src.getchannel("A") if frame.shape[2] == 4 else Image.fromarray(mask)
                        if mask is not None else None)
            recorded.clear()
            crop = ref_utils.crop_frame(np.array(black), None, intrinsic=K, openCV_pose=pose, image_size=S,
                                        keep_inplane=keep_inplane, virtual_bbox_size=vbs)
            M = recorded[0]
            _, inv = cv2.invert(M, flags=cv2.DECOMP_LU)
            normalised = img_transform(crop).numpy()
            # the crop as the model sees it is a function of the uint8 crop: check that here, store the uint8
            assert np.array_equal(normalised, (crop.astype(np.float32) / np.float32(255)) * 2 - np.float32(1))
            for k, v in dict(frame=np.array(fname), mask=np.zeros(0, np.uint8) if mask is None else mask, K=K, pose=pose,
                             vbs=np.float64(vbs), S=np.int64(S), keep_inplane=np.bool_(keep_inplane), M=M, inv=inv,
                             crop=crop).items():
                data[f"{name}__{k}"] = v
            summary[name] = {"S": S, "nonzero": int((crop > 0).any(-1).sum())}
    finally:
        ref_utils.cv2.getPerspectiveTransform = get_perspective
    data["cases"] = np.array([c[0] for c in all_cases])
    np.savez_compressed(os.path.join(out_dir, "crop.npz"), **data)
    return summary


def main():
    print(json.dumps(write_crop(), indent=1))


if __name__ == "__main__":
    sys.exit(main())
