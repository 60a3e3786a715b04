"""Time crop_frames (CUDA events, median of repeats): B in {1, 16, 64} crops of 720x540 RGB frames with one mask per
crop, and of 512x512 RGBA renders, to 256x256.  The frames and maps are on the device already; the host -> device
upload of a batch is timed on its own.  Beside it, the CPU reference pipeline per crop for scale: PIL's paste, the
warp (cv2.warpPerspective, as crop_frame calls it) and ToTensor / x*2-1, one crop at a time as a dataloader worker
runs it.

    python tools/crop_time.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nope_b200.crop import crop_frames, crop_transforms, forward_map   # noqa: E402
from oracle.crop_oracle import PRIMESENSE_K, SHAPENET_K               # noqa: E402

S = 256


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def scene(kind, B, rng):
    if kind == "rgb+mask":
        H, W, C, K, Z, vbs = 540, 720, 3, PRIMESENSE_K, (0.5, 1.0), 0.13
    else:
        H, W, C, K, Z, vbs = 512, 512, 4, SHAPENET_K, (1.0, 1.5), 1.0
    frames = rng.integers(0, 256, (B, H, W, C), dtype=np.uint8)
    masks = rng.integers(0, 2, (B, H, W), dtype=np.uint8) * 255 if C == 3 else None
    poses = np.stack([np.eye(4)] * B)
    poses[:, :3, 3] = np.stack([rng.uniform(-0.05, 0.05, B), rng.uniform(-0.05, 0.05, B), rng.uniform(*Z, B)], 1)
    return frames, masks, K, poses, vbs


def time_gpu(frames, masks, inv, reps):
    f, m, i = torch.from_numpy(frames), None if masks is None else torch.from_numpy(masks), torch.from_numpy(inv)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_up, t_k = [], []
    for r in range(reps + 2):
        ev[0].record()
        fd, md, idv = f.cuda(), None if m is None else m.cuda(), i.cuda()
        ev[1].record()
        crop_frames(fd, idv, S, masks=md)
        ev[2].record()
        torch.cuda.synchronize()
        if r >= 2:
            t_up.append(ev[0].elapsed_time(ev[1]))
            t_k.append(ev[1].elapsed_time(ev[2]))
    return float(np.median(t_k)), float(np.median(t_up))


def time_cpu(frames, masks, K, poses, vbs):
    """one crop, the reference's pipeline: paste, getPerspectiveTransform + warpPerspective, ToTensor, x*2-1"""
    import cv2
    from PIL import Image
    from torchvision import transforms
    tt = transforms.ToTensor()
    t0 = time.perf_counter()
    n = min(len(frames), 8)
    for b in range(n):
        src = Image.fromarray(frames[b])
        black = Image.new("RGB", src.size, (0, 0, 0))
        black.paste(src, mask=src.getchannel("A") if frames.shape[3] == 4 else Image.fromarray(masks[b]))
        M = forward_map(K, poses[b], vbs, S)
        tt(cv2.warpPerspective(np.asarray(black), M, (S, S))) * 2.0 - 1.0
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    name, pl = card()
    print(f"# {name}, power limit {pl}; crops to {S}x{S}; ms, median of {a.reps}")
    rng = np.random.default_rng(0)
    rows = []
    for kind in ("rgb+mask", "rgba"):
        for B in (1, 16, 64):
            frames, masks, K, poses, vbs = scene(kind, B, rng)
            inv = crop_transforms(K, poses, vbs, S)
            k_ms, up_ms = time_gpu(frames, masks, inv, a.reps)
            row = {"frames": "720x540 RGB + mask" if kind == "rgb+mask" else "512x512 RGBA", "B": B,
                   "kernel_ms": round(k_ms, 4), "kernel_us_per_crop": round(1e3 * k_ms / B, 2),
                   "upload_ms": round(up_ms, 3)}
            if B == 16:
                row["cpu_reference_ms_per_crop"] = round(time_cpu(frames, masks, K, poses, vbs), 2)
            rows.append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps({"card": name, "power_limit": pl, "rows": rows}))


if __name__ == "__main__":
    main()
