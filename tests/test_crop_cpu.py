"""CPU: full-frame crops without a device -- the numpy restatement of crop_warp_kernel (oracle/crop_oracle.py)
against the live reference pipeline (PIL paste, cv2.warpPerspective, torchvision) and against the unmodified
reference's crops (tests/golden/crop.npz), crop_transforms against the M the reference's crop_frame computes, the
weight table, the coordinate association, and the ABI's refusals and Python argument errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import crop_oracle as co


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "crop.npz")))


def _case(g, name):
    c = {k.split("__", 1)[1]: v for k, v in g.items() if k.startswith(name + "__")}
    c["frame"] = g["frame_" + str(c["frame"])]
    c["mask"] = None if c["mask"].size == 0 else c["mask"]
    return c


@pytest.fixture(scope="module")
def cases():
    pytest.importorskip("cv2")
    return co.seeded_cases()


# ------------------------------------------------------------------ the convention
def test_weight_table():
    """the float32 products times 32768 are exact, so every entry already sums to 32768 and equals the closed form
    32 (32 - fy or fy) (32 - fx or fx); the correction step never changes a weight"""
    tab = co.bilinear_table()
    closed = np.array([[(32 - i) * (32 - j), (32 - i) * j, i * (32 - j), i * j] for i in range(32) for j in range(32)])
    assert np.array_equal(tab, 32 * closed)
    assert (tab.sum(1) == 32768).all() and tab[0].tolist() == [32768, 0, 0, 0]


def test_div255_is_pils_paste():
    Image = pytest.importorskip("PIL.Image")
    v = np.arange(256, dtype=np.uint8)
    img = np.repeat(v[None, :, None], 256, 0).repeat(3, 2)            # every (value, mask) pair
    mask = np.repeat(v[:, None], 256, 1)
    black = Image.new("RGB", (256, 256))
    black.paste(Image.fromarray(img), mask=Image.fromarray(mask))
    assert np.array_equal(np.asarray(black), co.masked_frame(img, mask))


def _live(case):
    """the reference's pipeline run live: paste onto black, cv2.warpPerspective with crop_frame's M, ToTensor /
    Resize / x*2-1"""
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    transforms = pytest.importorskip("torchvision.transforms")
    frame, mask, S = case["frame"], case["mask"], int(case["S"])
    src = Image.fromarray(frame)
    black = Image.new("RGB", src.size, (0, 0, 0))
    black.paste(src, mask=src.getchannel("A") if frame.shape[2] == 4 else
                (Image.fromarray(mask) if mask is not None else None))
    u8 = cv2.warpPerspective(np.asarray(black), case["M"], (S, S))
    t = transforms.Compose([transforms.ToTensor(), transforms.Resize(S),
                            transforms.Lambda(lambda x: x * 2.0 - 1.0)])(u8)
    return u8, t.numpy()


@pytest.mark.parametrize("i", range(48))
def test_oracle_equals_live_pipeline(cases, i):
    c = cases[i]
    u8, ref = _live(c)
    ours = co.warp_u8(c["frame"], c["inv_map"], c["S"], c["mask"])
    assert np.array_equal(ours, u8), (c["name"], int((ours != u8).any(-1).sum()))
    assert np.array_equal(co.crop(c["frame"], c["inv_map"], c["S"], c["mask"]), ref), c["name"]


def test_seeded_cases_cover_the_ground(cases):
    S = {c["S"] for c in cases}
    kinds = {("rgba" if c["frame"].shape[2] == 4 else "binary" if c["mask"] is not None else "none") for c in cases}
    assert S == {256, 64, 17} and kinds == {"none", "binary", "rgba"}
    assert {c["keep_inplane"] for c in cases} == {False, True}
    scale = [float(c["name"].rsplit("/", 1)[1][:-1]) for c in cases]
    assert min(scale) < 0.5 and max(scale) > 2.0                       # magnified and minified
    frac = [(co.warp_u8(c["frame"], c["inv_map"], c["S"], c["mask"]) > 0).any(-1).mean() for c in cases]
    where = [c["name"].split("/")[1] for c in cases]
    assert all(f == 0 for f, w in zip(frac, where) if w == "outside")
    assert any(0.1 < f < 0.9 for f, w in zip(frac, where) if w == "partly")
    assert any(f > 0.9 for f, w in zip(frac, where) if w == "inside")
    assert any(c["frame"].shape[:2] == (251, 333) for c in cases)


def test_block_association(golden):
    """OpenCV sums (M0 xb + M1 y) + M2 per 64-column block, then + M0 (x - xb): in this crop pixel (100, 99) rounds
    to another 1/32 px row under the naive ((M0 x + M1 y) + M2) and changes value; the reference has the block's"""
    c = _case(golden, "block_assoc")
    Xb, Yb = co.fixed_coords(c["inv"], 256)
    Xn, Yn = co.fixed_coords(c["inv"], 256, block_w=256)
    differ = np.argwhere((Xb != Xn) | (Yb != Yn)).tolist()
    assert differ == [[100, 99]]
    block = co.warp_u8(c["frame"], c["inv"], 256)
    naive = co.warp_u8(c["frame"], c["inv"], 256, block_w=256)
    assert np.array_equal(block, c["crop"])
    assert np.argwhere((naive != c["crop"]).any(-1)).tolist() == [[100, 99]]
    cv2 = pytest.importorskip("cv2")
    assert np.array_equal(cv2.warpPerspective(c["frame"], c["M"], (256, 256)), block)


# ------------------------------------------------------------------ against the unmodified reference (fixture)
def test_oracle_reproduces_reference_crops(golden):
    names = [str(n) for n in golden["cases"]]
    assert len(names) == 8
    for name in names:
        c = _case(golden, name)
        assert np.array_equal(co.warp_u8(c["frame"], c["inv"], int(c["S"]), c["mask"]), c["crop"]), name
    assert (_case(golden, "outside")["crop"] == 0).all()
    part = (_case(golden, "partly_outside")["crop"] > 0).any(-1).mean()
    assert 0.1 < part < 0.9


@pytest.mark.parametrize("name", ["bop_upright", "bop_inplane", "shapenet_rgba", "shapenet_axis", "odd_frame",
                                  "partly_outside", "outside", "block_assoc"])
def test_crop_transforms_equal_reference_maps(golden, name):
    pytest.importorskip("cv2")
    from nope_b200.crop import crop_transforms, forward_map
    c = _case(golden, name)
    S, ki = int(c["S"]), bool(c["keep_inplane"])
    assert np.array_equal(forward_map(c["K"], c["pose"], float(c["vbs"]), S, ki), c["M"])
    inv = crop_transforms(c["K"], c["pose"], float(c["vbs"]), S, ki)
    assert inv.dtype == np.float64 and inv.shape == (1, 3, 3)
    assert np.array_equal(inv[0], c["inv"])


def test_fallback_branch():
    """an unrotated object on the optical axis: keep_inplane=False's `right` and `upper` are both zero and crop_frame
    falls back to the image axes, a box centred on the principal point"""
    pytest.importorskip("cv2")
    from nope_b200.crop import _corners, crop_transforms
    pose = np.eye(4)
    pose[2, 3] = 1.2
    c = _corners(co.SHAPENET_K, pose, 1.0, False)
    lo, hi = int(256 - 525 * 0.5 / 1.2), int(256 + 525 * 0.5 / 1.2)     # 37.25 and 474.75, truncated
    assert c.tolist() == [[lo, lo], [lo, hi], [hi, lo], [hi, hi]]
    assert np.isfinite(crop_transforms(co.SHAPENET_K, pose, 1.0, 64)).all()
    # keep_inplane=True needs y = z = 0 for its fallback, an object at Z = 0, which is refused
    pose[2, 3] = 0.0
    for ki in (False, True):
        with pytest.raises(ValueError, match="Z > 0"):
            crop_transforms(co.SHAPENET_K, pose, 1.0, 64, keep_inplane=ki)


def test_crop_transforms_batching_and_errors():
    pytest.importorskip("cv2")
    from nope_b200.crop import crop_transforms
    K = co.PRIMESENSE_K
    poses = np.stack([np.eye(4)] * 3)
    poses[:, :3, 3] = [[0.01, 0.0, 0.6], [0.0, 0.02, 0.7], [-0.03, 0.01, 0.5]]
    batched = crop_transforms(np.stack([K] * 3), poses, [0.1, 0.12, 0.1], 64, keep_inplane=True)
    one = np.stack([crop_transforms(K, p, v, 64, keep_inplane=True)[0] for p, v in zip(poses, [0.1, 0.12, 0.1])])
    assert np.array_equal(batched, one)
    assert crop_transforms(torch.from_numpy(K), torch.from_numpy(poses), 0.1).shape == (3, 3, 3)
    for args in [(K[:2], poses, 0.1), (K, poses[:, :3], 0.1), (np.stack([K] * 2), poses, 0.1), (K, poses, [0.1] * 2),
                 (K, poses, 0.0), (K, poses, float("nan")), (K, poses, np.ones((3, 1)))]:
        with pytest.raises(ValueError):
            crop_transforms(*args)
    for S in (0, 4097, 2.5):
        with pytest.raises(ValueError):
            crop_transforms(K, poses, 0.1, S)
    behind = poses.copy()
    behind[1, 2, 3] = -0.5
    with pytest.raises(ValueError, match="Z > 0"):
        crop_transforms(K, behind, 0.1)


# ------------------------------------------------------------------ ABI
P = C.c_void_p(256)
_A = dict(fr=P, F=2, H=540, W=720, C=3, mk=None, fi=None, inv=P, B=2, S=256, o=P)


@pytest.mark.parametrize("bad,needle", [
    (dict(fr=None), "null"), (dict(inv=None), "null"), (dict(o=None), "null"),
    (dict(F=0), "F and B"), (dict(B=0, F=0), "F and B"), (dict(B=0), "F and B"), (dict(B=65536, fi=P), "B must"),
    (dict(H=0), "H and W"), (dict(W=0), "H and W"), (dict(H=16385), "H and W"), (dict(W=16385), "H and W"),
    (dict(S=0), "S must"), (dict(S=4097), "S must"), (dict(C=1), "C must"), (dict(C=5), "C must"),
    (dict(C=4, mk=P), "mask"), (dict(F=3), "frame_idx")])
def test_crop_refusals(bad, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    a = {**_A, **bad}
    assert lib.nope_crop_frames(a["fr"], a["F"], a["H"], a["W"], a["C"], a["mk"], a["fi"], a["inv"], a["B"], a["S"],
                                a["o"], None) != 0
    assert needle in lib.nope_last_error().decode()


def test_python_argument_errors():
    """every malformed argument raises before any device work (these run without a GPU)"""
    from nope_b200.crop import crop_frames
    fr = torch.zeros(2, 6, 8, 3, dtype=torch.uint8)
    inv = torch.eye(3, dtype=torch.float64).repeat(2, 1, 1)
    bad = [dict(frames=fr.float()), dict(frames=fr[0]), dict(frames=torch.zeros(2, 6, 8, 2, dtype=torch.uint8)),
           dict(frames=torch.zeros(0, 6, 8, 3, dtype=torch.uint8)),
           dict(frames=torch.zeros(1, 16385, 1, 3, dtype=torch.uint8)),
           dict(inv_maps=inv.float()), dict(inv_maps=inv[:, :2]), dict(inv_maps=inv[:1]),
           dict(image_size=0), dict(image_size=4097), dict(image_size=1.5),
           dict(masks=torch.zeros(2, 6, 8)), dict(masks=torch.zeros(2, 6, 9, dtype=torch.uint8)),
           dict(masks=torch.zeros(1, 6, 8, dtype=torch.uint8)),
           dict(frames=torch.zeros(2, 6, 8, 4, dtype=torch.uint8), masks=torch.zeros(2, 6, 8, dtype=torch.uint8)),
           dict(frame_idx=torch.zeros(3, dtype=torch.int64)), dict(frame_idx=torch.zeros(2)),
           dict(frames=fr[:1])]
    for kw in bad:
        args = {"frames": fr, "inv_maps": inv, "image_size": 16, **kw}
        with pytest.raises(ValueError):
            crop_frames(**args)
