"""CPU: pose tracking (DESIGN.md section 26) without a device.  The numpy oracle of track_seed_kernel reconstructs
each prior from its centre, picks the template a brute-force search over the roll picks, and maps non-finite priors
to (I, 0, (1, 0)); the ABI declares and binds nope_track_seeds and refuses bad arguments before any CUDA call; every
refusal of the dict seeds of refine_inplane, track_inplane, track_pose_frames and PoseTracker fires before any device
work."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import track_oracle as to


@pytest.fixture(scope="module")
def grid():
    from nope_b200.poses import icosphere_object_rotations
    return icosphere_object_rotations(1)                                  # 162 poses


def test_centres_reconstruct_the_prior(grid):
    rng = np.random.default_rng(0)
    Rc = to.random_rotations(300, rng)
    D, seed, cs = to.track_seeds(Rc, grid)
    assert D.dtype == np.float32 and seed.dtype == np.int32 and cs.dtype == np.float32
    assert ((seed >= 0) & (seed < len(grid))).all()
    err = np.abs(to.compose(D, seed, cs, grid) - Rc).max()
    assert err <= 1e-6, err                                               # fp32 rounding of D and (c, s)
    # the residual turns about an axis in the xy plane: its z component D10 - D01 vanishes
    assert np.abs(D[:, 1, 0] - D[:, 0, 1]).max() <= 1e-6
    assert np.abs(np.hypot(cs[:, 0].astype(np.float64), cs[:, 1]) - 1).max() <= 1e-7


def test_priors_on_grid_poses_recover_template_and_roll(grid):
    rng = np.random.default_rng(1)
    n = rng.integers(0, len(grid), 50)
    beta = rng.uniform(-180, 180, 50)
    Rc = np.stack([to.rz(b) @ grid[i] for b, i in zip(beta, n)])
    D, seed, cs = to.track_seeds(Rc, grid)
    assert np.array_equal(seed, n)
    assert np.abs(D - np.eye(3, dtype=np.float32)).max() <= 1e-6
    got = np.degrees(np.arctan2(cs[:, 1].astype(np.float64), cs[:, 0]))
    assert np.abs((got - beta + 180) % 360 - 180).max() <= 1e-4


def test_same_template_as_a_brute_force_roll_search(grid):
    """the best trace over rolls at 0.01 degree steps picks the oracle's template, or one whose brute-force score is
    within what that step can resolve (r (1 - cos 0.005 deg) <= 8e-9)"""
    rng = np.random.default_rng(2)
    Rc = to.random_rotations(40, rng)
    _, seed, _ = to.track_seeds(Rc, grid)
    M = to.residuals(Rc, grid)
    a, b, _, _ = to.scores(M)
    rho = np.deg2rad(np.arange(0, 360, 0.01))
    c, s = np.cos(rho), np.sin(rho)
    for h in range(len(Rc)):
        bf = (a[h][:, None] * c[None] + b[h][:, None] * s[None]).max(axis=1) + M[h, :, 2, 2]
        assert seed[h] == int(np.argmax(bf)) or bf[seed[h]] >= bf.max() - 1e-8, h


def test_non_finite_priors_ties_and_nan_grid_rows(grid):
    rng = np.random.default_rng(3)
    Rc = to.random_rotations(4, rng)
    Rc[1, 2, 0] = np.nan
    Rc[2, 0, 1] = np.inf
    D, seed, cs = to.track_seeds(Rc, grid)
    for h in (1, 2):
        assert seed[h] == 0 and np.array_equal(D[h], np.eye(3, dtype=np.float32)) and np.array_equal(cs[h], [1, 0])
    # a NaN grid row is never chosen; duplicated rows tie and the lowest index wins
    T = np.concatenate([grid[:10], grid[:10]])
    T[3] = np.nan
    prior = np.stack([to.rz(7.0) @ grid[3], to.rz(-20.0) @ grid[5]])
    _, s2, _ = to.track_seeds(prior, T)
    assert s2[0] == 13 and s2[1] == 5
    _, s3, cs3 = to.track_seeds(to.random_rotations(3, rng), np.full((4, 3, 3), np.nan))
    assert (s3 == 0).all() and (cs3 == [1, 0]).all()


def test_abi_declares_binds_and_refuses():
    from nope_b200 import _lib
    lib = _lib.load()
    assert "nope_track_seeds" in _lib.SIGNATURES and hasattr(lib, "nope_track_seeds")
    p = C.c_void_p(8)
    assert lib.nope_track_seeds(None, 1, p, 1, p, p, p, None) != 0
    assert b"null" in lib.nope_last_error()
    for H, N in ((0, 5), (3, 0), (-1, 5)):
        assert lib.nope_track_seeds(p, H, p, N, p, p, p, None) != 0
        assert b"H and N" in lib.nope_last_error()


# ------------------------------------------------------------------ refusals before device work
@pytest.fixture
def no_device(monkeypatch):
    """every native call and the frame crops fail loudly: a refusal must come first"""
    from nope_b200 import _lib, crop, inplane_refine

    def boom(*a, **kw):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(crop, "frame_crops", boom)
    monkeypatch.setattr(inplane_refine, "row_pairs", boom)
    return boom


def _engine(channels=8):
    def sweep(*a, **kw):
        raise AssertionError("device work before the refusal")
    cls = type("UNet", (), {})
    e = cls()
    e.channels, e.precision, e.device = channels, "fp16", torch.device("cpu")
    e.encoder = types.SimpleNamespace(precision="split", latent_dim=channels, encode_image_rotated=sweep,
                                      encode_image=sweep)
    e.sweep = e.set_metric = sweep
    return e


def _refiner(grid, A=4, steps=2):
    from nope_b200.inplane_refine import InplaneRefiner
    return InplaneRefiner(torch.from_numpy(grid), A, steps)


def test_dict_seed_refusals(grid, no_device):
    from nope_b200.inplane_refine import refine_inplane
    e, ref = _engine(), _refiner(grid)
    B, N, keep = 2, len(grid), 2
    rf, q, rel = torch.zeros(B, 8, 32, 32), torch.zeros(B, 3, 256, 256), torch.zeros(B, N, 6)
    lat = torch.zeros(B, keep, 8, 32, 32)
    good = {"D": torch.zeros(B, keep, 3, 3), "seed": torch.zeros(B, keep, dtype=torch.int64),
            "cossin": torch.zeros(B, keep, 2)}
    for bad, needle in ((dict(good, extra=good["D"]), "dict of tensors"), ({"D": good["D"]}, "dict of tensors"),
                        (dict(good, seed=good["seed"].float()), "integer"),
                        (dict(good, D=good["D"].double()), "float32"),
                        (dict(good, cossin=good["cossin"].double()), "float32"),
                        (dict(good, D=good["D"][:, :1]), "centre seeds"),
                        (dict(good, cossin=good["cossin"][..., :1]), "centre seeds"),
                        (dict(good, seed=good["seed"][None]), "centre seeds"),
                        (dict(good, seed=good["seed"][:, :0], D=good["D"][:, :0], cossin=good["cossin"][:, :0]),
                         "centre seeds")):
        with pytest.raises(ValueError, match=needle):
            refine_inplane(e, e.encoder, rf, q, rel, bad, lat, ref, k=3)
    big = {"D": torch.zeros(B, 17, 3, 3), "seed": torch.zeros(B, 17, dtype=torch.int32),
           "cossin": torch.zeros(B, 17, 2)}
    with pytest.raises(ValueError, match="keep must be"):
        refine_inplane(e, e.encoder, rf, q, rel, big, torch.zeros(B, 17, 8, 32, 32), ref, k=3)
    with pytest.raises(ValueError, match="k must be"):
        refine_inplane(e, e.encoder, rf, q, rel, good, lat, ref, k=65)
    with pytest.raises(ValueError, match="seed_latents"):
        refine_inplane(e, e.encoder, rf, q, rel, good, lat[:, :1], ref, k=3)
    with pytest.raises(ValueError, match="query"):
        refine_inplane(e, e.encoder, rf, q[:, None, :, :4], rel, good, lat, ref, k=3)
    with pytest.raises(AssertionError, match="device work"):                   # the arguments are fine
        refine_inplane(e, e.encoder, rf, q, rel, good, lat, ref, k=3)


def test_track_inplane_and_seed_centres_refusals(grid, no_device):
    from nope_b200 import _lib
    from nope_b200.track import seed_centres, track_inplane
    e, ref = _engine(), _refiner(grid)
    B, N = 2, len(grid)
    rf, q, rel = torch.zeros(B, 8, 32, 32), torch.zeros(B, 3, 256, 256), torch.zeros(B, N, 6)
    R = torch.eye(3, dtype=torch.float64).repeat(B, 2, 1, 1)
    for args, needle in (((rf, q[:, :2], rel, R), "crops"), ((rf[:1], q, rel, R), "ref_feat"),
                         ((rf, q, rel, R[:1]), "R_prior"), ((rf, q, rel, R[..., :2]), "R_prior"),
                         ((rf, q, rel, R[:, :0]), "R_prior"), ((rf, q, rel, R.repeat(1, 9, 1, 1)), "at most 16"),
                         ((rf, q, rel, R.half()), "float32 or float64"), ((rf, q, rel[:, :5], R), "refiner's grid"),
                         ((rf, q, rel[:1], R), "references")):
        with pytest.raises(ValueError, match=needle):
            track_inplane(e, e.encoder, *args, ref, k=3)
    with pytest.raises(ValueError, match="k must be"):
        track_inplane(e, e.encoder, rf, q, rel, R, ref, k=0)
    with pytest.raises(ValueError, match="exceeds"):
        track_inplane(e, e.encoder, rf, q, rel, R[:, :1], ref, k=28)
    with pytest.raises(ValueError, match="refiner"):
        track_inplane(e, e.encoder, rf, q, rel, R, object(), k=3)
    with pytest.raises(ValueError, match="refiner"):
        seed_centres(R, object())
    with pytest.raises(_lib.NopeError, match="CUDA"):
        seed_centres(R, ref)


def _frames_model(grid):
    from nope_b200.bank import TemplateBank, engine_descriptor
    from nope_b200.model import PoseConditional
    e = _engine()
    m = PoseConditional(e)
    for i in (4, 9):
        m.tless_cad[i] = object()
        m.bop_models[i] = {"diameter": 100.0}
    g = torch.Generator().manual_seed(0)
    n = len(grid)
    tp = torch.from_numpy(grid)
    bank = TemplateBank([4, 9], torch.randn(2, n, 8, 32, 32, generator=g), torch.randn(2, 8, 32, 32, generator=g),
                        torch.randn(2, n, 6, generator=g), tp, engine_descriptor(e))
    return m, bank


def test_track_pose_frames_refusals(grid, no_device):
    m, bank = _frames_model(grid)
    ref = _refiner(grid)
    frames, masks = torch.zeros(2, 8, 8, 3, dtype=torch.uint8), torch.zeros(2, 8, 8, dtype=torch.uint8)
    K = torch.eye(3, dtype=torch.float64)
    R = torch.eye(3, dtype=torch.float64).repeat(2, 2, 1, 1)
    N = len(grid)
    refs = (torch.zeros(1, 3, 256, 256), torch.zeros(1, N, 6))
    cases = [((frames, masks, K, [4, 9], R, ref), dict(bank=bank, refine="depth"), "refine"),
             ((frames, masks, K, [4, 9], R, ref), dict(bank=bank, occluders="others"), "occluders"),
             ((frames, masks, K, [4], R, ref), dict(bank=bank), "obj_ids for"),
             ((frames, masks, K, [4, 7], R, ref), dict(bank=bank), "models_info"),
             ((frames, masks, K, [4, 9], R, ref), dict(), "or a bank"),
             ((frames, masks, K, [4, 9], R, ref), dict(bank=bank, reference=refs[0]), "not both"),
             ((frames, masks, K, [4, 9], R, ref), dict(reference=torch.zeros(3, 3, 256, 256),
                                                       all_relativeR=refs[1]), "reference"),
             ((frames, masks, K, [4, 9], R, object()), dict(bank=bank), "refiner"),
             ((frames, masks, K, [4, 9], R, _refiner(grid[:42])), dict(bank=bank), "pose grid"),
             ((frames, masks, K, [4, 9], R[:1], ref), dict(bank=bank), "R_prior"),
             ((frames, masks, K, [4, 9], R[..., :2], ref), dict(bank=bank), "R_prior"),
             ((frames, masks, K, [4, 9], R.repeat(1, 9, 1, 1), ref), dict(bank=bank), "at most 16"),
             ((frames, masks, K, [4, 9], R, ref), dict(bank=bank, k=0), "k must be"),
             ((frames, masks, K, [4, 9], R[:, :1], ref), dict(bank=bank, k=28), "exceeds"),
             ((frames, masks, K, [4, 9], R, ref), dict(reference=refs[0], all_relativeR=torch.zeros(2, N, 6)),
              "references"),
             ((frames, masks, K, [4, 9], R, ref), dict(reference=refs[0], all_relativeR=refs[1],
                                                       template_poses=torch.from_numpy(grid).flip(0)),
              "refiner's grid")]
    for args, kw, needle in cases:
        with pytest.raises(ValueError, match=needle):
            m.track_pose_frames(*args, **kw)
    m.testing_config.similarity_metric = "dot"
    with pytest.raises(ValueError, match="similarity_metric"):
        m.track_pose_frames(frames, masks, K, [4, 9], R, ref, bank=bank)
    m.testing_config.similarity_metric = "l2"
    m.dist = object()
    with pytest.raises(NotImplementedError, match="does not shard"):
        m.track_pose_frames(frames, masks, K, [4, 9], R, ref, bank=bank)
    m.dist = None
    with pytest.raises(AssertionError, match="device work"):                    # the arguments are fine
        m.track_pose_frames(frames, masks, K, [4, 9], R, ref, bank=bank)
    with pytest.raises(AssertionError, match="device work"):
        m.track_pose_frames(frames, masks, K, [4, 9], R, ref, reference=refs[0], all_relativeR=refs[1],
                            template_poses=torch.from_numpy(grid))


def test_pose_tracker_refusals(grid, no_device):
    from nope_b200.track import PoseTracker
    m, bank = _frames_model(grid)
    ref = _refiner(grid)
    for kw, needle in ((dict(keep=3, k=2), "at least keep"), (dict(keep=17, k=20), "keep must be"),
                       (dict(k=65), "k must be"), (dict(min_iou=1.5), "min_iou"), (dict(min_iou=True), "min_iou"),
                       (dict(refine="depth"), "refine"), (dict(occluders=torch.zeros(2, 8, 8)), "occluders")):
        with pytest.raises(ValueError, match=needle):
            PoseTracker(m, bank, ref, **kw)
    with pytest.raises(ValueError, match="TemplateBank"):
        PoseTracker(m, object(), ref)
    with pytest.raises(ValueError, match="refiner"):
        PoseTracker(m, bank, object())
    with pytest.raises(ValueError, match="pose grid"):
        PoseTracker(m, bank, _refiner(grid[::-1].copy()))
    m.dist = object()
    with pytest.raises(NotImplementedError, match="does not shard"):
        PoseTracker(m, bank, ref)
    m.dist = None
    tr = PoseTracker(m, bank, ref, keep=2, k=3)
    frames, masks = torch.zeros(2, 8, 8, 3, dtype=torch.uint8), torch.zeros(2, 8, 8, dtype=torch.uint8)
    K = torch.eye(3, dtype=torch.float64)
    with pytest.raises(ValueError, match="distinct track_ids"):
        tr.step(frames, masks, K, [4, 9], [1, 1])
    with pytest.raises(ValueError, match="distinct track_ids"):
        tr.step(frames, masks, K, [4, 9], [1])
    with pytest.raises(ValueError, match="masks"):
        tr.step(frames, masks[:1], K, [4, 9], [1, 2])
    with pytest.raises(ValueError, match="K"):
        tr.step(frames, masks, np.zeros((3, 3, 3)), [4, 9], [1, 2])
    # a known track whose object changes: refused before the search or the tracking of any row
    tr.tracks = {1: (4, torch.eye(3, dtype=torch.float64).repeat(2, 1, 1)), 2: (9, None)}
    with pytest.raises(ValueError, match=r"track ids \[2\] changed obj_id"):
        tr.step(frames, masks, K, [4, 4], [1, 2])
    assert set(tr.tracks) == {1, 2}                                             # nothing forgotten by a refusal
    with pytest.raises(AssertionError, match="device work"):                    # the arguments are fine
        tr.step(frames, masks, K, [4, 9], [1, 3])
