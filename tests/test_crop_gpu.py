"""GPU: full-frame crops.  crop_warp_kernel against the numpy oracle bit for bit on every CPU-test case and against the
unmodified reference's crops (tests/golden/crop.npz); checks that need no oracle (integer translations copy, the first
pixel sits at the box's first corner, black crops outside the frame and for out-of-range frame indices); batching,
shared frames and no host synchronisation; predict_pose and predict_pose_inplane on the crops."""
import os

import numpy as np
import pytest
import torch

from _util import no_host_sync
from oracle import crop_oracle as co
from oracle import inputs

pytestmark = pytest.mark.gpu


def _crop(frame, inv, S, mask=None):
    from nope_b200.crop import crop_frames
    f = torch.from_numpy(np.ascontiguousarray(frame))[None]
    m = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask))[None]
    out = crop_frames(f, torch.from_numpy(np.asarray(inv, dtype=np.float64)).reshape(1, 3, 3), S, masks=m)
    return out[0].cpu().numpy()


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.int32), np.asarray(b, dtype=np.float32).view(np.int32))


@pytest.fixture(scope="module")
def cases():
    return co.seeded_cases()


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "crop.npz")))


def _case(g, name):
    c = {k.split("__", 1)[1]: v for k, v in g.items() if k.startswith(name + "__")}
    c["frame"] = g["frame_" + str(c["frame"])]
    c["mask"] = None if c["mask"].size == 0 else c["mask"]
    return c


# ------------------------------------------------------------------ kernel vs oracle and reference
def test_kernel_equals_oracle_on_every_cpu_case(cases):
    for c in cases:
        out = _crop(c["frame"], c["inv_map"], c["S"], c["mask"])
        assert out.shape == (3, c["S"], c["S"])
        assert _same(out, co.crop(c["frame"], c["inv_map"], c["S"], c["mask"])), c["name"]


def test_kernel_equals_reference_crops(golden):
    for name in golden["cases"]:
        c = _case(golden, str(name))
        out = _crop(c["frame"], c["inv"], int(c["S"]), c["mask"])
        assert _same(out, co.normalise(c["crop"])), name


# ------------------------------------------------------------------ without the oracle
def test_integer_translation_copies():
    rng = np.random.default_rng(5)
    frame = rng.integers(0, 256, (70, 90, 3), dtype=np.uint8)
    mask = rng.integers(0, 256, (70, 90), dtype=np.uint8)
    for tx, ty, S in ((0, 0, 64), (13, 5, 40), (26, 6, 17)):
        inv = np.array([[1.0, 0, tx], [0, 1.0, ty], [0, 0, 1.0]])
        want = frame[ty:ty + S, tx:tx + S].astype(np.float32)
        assert _same(_crop(frame, inv, S), np.moveaxis(want / np.float32(255) * 2 - 1, -1, 0))
        m = mask[ty:ty + S, tx:tx + S, None].astype(np.int64)
        pasted = (((frame[ty:ty + S, tx:tx + S] * m + 128) >> 8) + frame[ty:ty + S, tx:tx + S] * m + 128) >> 8
        assert _same(_crop(frame, inv, S, mask), np.moveaxis(pasted.astype(np.float32) / np.float32(255) * 2 - 1,
                                                             -1, 0))


def test_first_pixel_is_the_first_corner(golden):
    """crop_frame maps corner w1 (truncated to int32) to the crop's (0, 0): that pixel is the masked source pixel"""
    from nope_b200.crop import _corners, crop_transforms
    for name in ("bop_upright", "bop_inplane", "shapenet_axis", "odd_frame"):         # w1 inside the frame
        c = _case(golden, name)
        S, ki = int(c["S"]), bool(c["keep_inplane"])
        u, v = _corners(c["K"], c["pose"], float(c["vbs"]), ki)[0]
        assert 0 <= u < c["frame"].shape[1] and 0 <= v < c["frame"].shape[0], name
        out = _crop(c["frame"], crop_transforms(c["K"], c["pose"], float(c["vbs"]), S, ki)[0], S, c["mask"])
        src = co.masked_frame(c["frame"], c["mask"])[v, u].astype(np.float32)
        assert _same(out[:, 0, 0], src / np.float32(255) * 2 - 1), name


def test_outside_and_bad_frame_index_are_black():
    from nope_b200.crop import crop_frames
    rng = np.random.default_rng(6)
    frames = torch.from_numpy(rng.integers(0, 256, (2, 40, 50, 3), dtype=np.uint8)).cuda()
    inv = torch.tensor([[1.0, 0, 3], [0, 1.0, 2], [0, 0, 1.0]], dtype=torch.float64).repeat(4, 1, 1)
    inv[3, 0, 2] = 1000.0                                                # a crop entirely beside the frame
    idx = torch.tensor([0, 2, 1, 0], dtype=torch.int32)
    out = crop_frames(frames, inv, 24, frame_idx=idx)
    assert (out[1] == -1).all() and (out[3] == -1).all()
    alone = [crop_frames(frames[i:i + 1], inv[b:b + 1], 24) for b, i in ((0, 0), (2, 1))]
    assert torch.equal(out[0], alone[0][0]) and torch.equal(out[2], alone[1][0])
    for bad in (-1, 2, 1 << 40):
        assert (crop_frames(frames, inv[:1], 24, frame_idx=torch.tensor([bad]))[0] == -1).all()


def test_shared_frames_and_batching():
    from nope_b200.crop import crop_frames, crop_transforms
    rng = np.random.default_rng(7)
    frames = torch.from_numpy(rng.integers(0, 256, (2, 540, 720, 3), dtype=np.uint8))
    poses = np.stack([np.eye(4)] * 5)
    poses[:, :3, 3] = [[0.01, 0.0, 0.6], [0.05, 0.02, 0.7], [-0.03, 0.01, 0.5], [0.0, -0.04, 0.8], [0.1, 0.0, 0.9]]
    inv = torch.from_numpy(crop_transforms(co.PRIMESENSE_K, poses, 0.12, 64))
    masks = torch.from_numpy(rng.integers(0, 256, (5, 540, 720), dtype=np.uint8))
    idx = torch.tensor([0, 1, 1, 0, 1])
    shared = crop_frames(frames, inv, 64, masks=masks, frame_idx=idx)
    dup = crop_frames(frames[idx], inv, 64, masks=masks)
    assert torch.equal(shared, dup)
    for b in range(5):
        one = crop_frames(frames[idx[b]][None], inv[b:b + 1], 64, masks=masks[b:b + 1])
        assert torch.equal(one[0], shared[b])
    dev = crop_frames(frames.cuda(), inv.cuda(), 64, masks=masks.cuda(), frame_idx=idx.cuda())
    assert dev.device.type == "cuda" and torch.equal(dev, shared)


def test_no_host_synchronisation():
    from nope_b200.crop import crop_frames
    frames = torch.randint(0, 256, (3, 120, 160, 4), dtype=torch.uint8, device="cuda")
    inv = torch.eye(3, dtype=torch.float64, device="cuda").repeat(2, 1, 1)
    idx = torch.tensor([2, 0], device="cuda")
    crop_frames(frames, inv, 32, frame_idx=idx)                            # warm-up: library load
    with no_host_sync():
        out = crop_frames(frames, inv, 32, frame_idx=idx)
    assert out.shape == (2, 3, 32, 32)


# ------------------------------------------------------------------ end to end
def test_predict_pose_on_crops(gpu_model, golden):
    """the model sees the kernel's crops exactly as it sees the oracle's: the same poses and scores"""
    from nope_b200.crop import crop_frames
    q, r = _case(golden, "bop_upright"), _case(golden, "bop_inplane")
    frames = torch.from_numpy(np.stack([q["frame"], r["frame"]]))
    masks = torch.from_numpy(np.stack([q["mask"], r["mask"]]))
    # 256 x 256 crops of the same two boxes
    from nope_b200.crop import crop_transforms
    inv = torch.from_numpy(np.concatenate([crop_transforms(q["K"], q["pose"], float(q["vbs"]), 256, False),
                                           crop_transforms(r["K"], r["pose"], float(r["vbs"]), 256, True)]))
    crops = crop_frames(frames, inv, 256, masks=masks)
    oracle = torch.from_numpy(co.crop_frames(frames.numpy(), inv.numpy(), 256, masks=masks.numpy()))
    assert torch.equal(crops.cpu(), oracle)
    poses, tposes = inputs.make_pose_batch("level0_upper", batch=1, n=6)
    a = gpu_model.predict_pose(crops[:1], crops[1:], poses.cuda(), tposes, k=5)
    b = gpu_model.predict_pose(oracle[:1].cuda(), oracle[1:].cuda(), poses.cuda(), tposes, k=5)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    R, n, ang, sim = gpu_model.predict_pose_inplane(crops[1:], crops[:1], poses.cuda(), tposes, k=3, angles=8)
    assert R.shape == (1, 3, 3, 3) and sim.shape == (1, 8, 6) and torch.isfinite(sim).all()
