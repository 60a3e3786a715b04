"""CPU: searches under occlusion (DESIGN.md section 27) without a device -- the identities of the visibility and score
oracle, the argument checks of the five C ABI entry points in the library, and the refusals of the Python layer
before any device work."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import visibility_oracle as vo

CL = 4


def _hidden(seed, B=2, p=0.002, S=256):
    rng = np.random.default_rng(seed)
    h = (rng.random((B, S, S)) < p).astype(np.uint8)
    h[:, 40:90, 100:180] = 1                                       # one solid region besides the scattered pixels
    return h


@pytest.mark.parametrize("seed", [0, 1])
def test_identity_roll_is_the_block_max(seed):
    h = _hidden(seed)
    V = vo.latent_visibility(h, [0, 1], [[1.0, 0.0], [1.0, 0.0]])
    for b in range(2):
        pooled = h[b].reshape(32, 8, 32, 8).max(axis=(1, 3))
        assert np.array_equal(V[b], (pooled == 0).astype(np.uint8))


def test_quarter_turns_permute_the_map():
    h = _hidden(7, B=1)
    base = vo.latent_visibility(h, [0], [[1.0, 0.0]])[0]
    for k, cs in ((1, (0.0, 1.0)), (2, (-1.0, 0.0)), (3, (0.0, -1.0))):
        assert np.array_equal(vo.rolled_hidden(h[0], *cs), np.rot90(h[0] != 0, k))
        assert np.array_equal(vo.latent_visibility(h, [0], [cs])[0], np.rot90(base, k))


def test_out_of_range_image_is_all_visible():
    h = np.ones((1, 256, 256), np.uint8)
    V = vo.latent_visibility(h, [-1, 1, 0], [[1.0, 0.0]] * 3)
    assert V[0].all() and V[1].all() and not V[2].any()


def test_crop_hidden_reads_only_weighted_taps():
    from oracle import crop_oracle
    case = crop_oracle.seeded_cases(n=1)[0]
    H, W = case["frame"].shape[:2]
    occ = np.zeros((1, H, W), np.uint8)
    assert not vo.crop_hidden(occ, case["inv_map"][None]).any()
    occ[0] = 1
    full = vo.crop_hidden(occ, case["inv_map"][None])
    # every crop pixel whose sample lands inside the frame is hidden, exactly those the warp reads
    X, Y = crop_oracle.fixed_coords(case["inv_map"], 256)
    sx, sy = X >> 5, Y >> 5
    assert full[0][(sx >= 0) & (sx < W - 1) & (sy >= 0) & (sy < H - 1)].all()


def _rows(seed, N=6, hw=1024):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(CL, hw, generator=g, dtype=torch.float64), torch.randn(N, CL, hw, generator=g,
                                                                               dtype=torch.float64)


@pytest.mark.parametrize("metric", ["l2", "cosine", "cosine_occlusion"])
def test_all_visible_scores_are_the_unweighted_scores(metric):
    q, t = _rows(0)
    got = vo.scores(q.numpy(), t.numpy(), np.ones(1024, np.uint8), metric)
    if metric == "l2":
        ref = -((q[None] - t) ** 4).sum(1).sqrt().sum(1)
    elif metric == "cosine":
        ref = torch.nn.functional.cosine_similarity(q.reshape(1, -1), t.reshape(t.shape[0], -1), eps=1e-8)
    else:
        per = torch.nn.functional.cosine_similarity(q[None], t, dim=1, eps=1e-8)
        ref = torch.where(per > 0.2, per, torch.zeros_like(per)).mean(1)
    np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12, atol=1e-12)


def test_substitution_identity():
    """the l2 score over the visible pixels is f times the unweighted l2 of a query whose hidden latents are the
    template's own"""
    q, t = _rows(1)
    rng = np.random.default_rng(1)
    vis = (rng.random(1024) < 0.3).astype(np.uint8)
    f = 1024 / vis.sum()
    got = vo.scores(q.numpy(), t.numpy(), vis, "l2")
    hid = torch.from_numpy(vis == 0)
    for n in range(t.shape[0]):
        qs = torch.where(hid[None], t[n], q)
        unweighted = -((qs - t[n]) ** 4).sum(0).sqrt().sum()
        np.testing.assert_allclose(got[n], f * float(unweighted), rtol=1e-12)
    assert np.isnan(vo.scores(q.numpy(), t.numpy(), np.zeros(1024, np.uint8), "l2")).all()


# ------------------------------------------------------------------ the C ABI, before any CUDA call
def _fake():
    return C.c_void_p(256)       # never dereferenced: every call below fails its argument checks first


def _lib():
    from nope_b200 import _lib
    return _lib.load()


def _err():
    return _lib().nope_last_error().decode()


def test_entry_points_are_declared_and_bound():
    from nope_b200 import _lib as L
    for name in ("nope_crop_hidden", "nope_latent_visibility", "nope_unet_sweep_visible", "nope_ldm_sweep_visible",
                 "nope_score_topk_visible"):
        assert name in L.SIGNATURES and hasattr(_lib(), name)
    assert _lib().nope_abi_version() == 3


def test_crop_hidden_refusals():
    def call(null=None, H=480, W=640, B=2, S=256):
        p = [_fake() for _ in range(3)]
        if null is not None:
            p[null] = None
        return _lib().nope_crop_hidden(p[0], H, W, p[1], B, S, p[2], None)
    for null in range(3):
        assert call(null=null) == -1 and "null" in _err()
    for kw, word in (({"B": 0}, "B must"), ({"B": 65536}, "B must"), ({"H": 0}, "H and W"), ({"W": 16385}, "H and W"),
                     ({"S": 250}, "S must"), ({"S": 128}, "S must"), ({"S": 0}, "S must")):
        assert call(**kw) == -1 and word in _err(), kw


def test_latent_visibility_refusals():
    def call(null=None, B=2, S=256, P=3):
        p = [_fake() for _ in range(4)]
        if null is not None:
            p[null] = None
        return _lib().nope_latent_visibility(p[0], B, S, p[1], p[2], P, p[3], None)
    for null in range(4):
        assert call(null=null) == -1 and "null" in _err()
    for kw, word in (({"B": 0}, "B must"), ({"S": 257}, "S must"), ({"S": 512}, "S must"), ({"P": 0}, "P (pairs)"),
                     ({"P": 2 ** 30}, "P (pairs)")):
        assert call(**kw) == -1 and word in _err(), kw


@pytest.mark.parametrize("engine", ["unet", "ldm"])
def test_sweep_visible_refusals(engine):
    fn = getattr(_lib(), f"nope_{engine}_sweep_visible")
    p = [_fake() for _ in range(8)]
    # a null query or visible map is refused before the engine is looked at
    assert fn(p[0], p[1], p[2], 1, 10, None, 1, p[3], None, p[4], 0, None, None, 0, None) == -1 and "null" in _err()
    assert fn(p[0], p[1], p[2], 1, 10, p[3], 1, None, None, p[4], 0, None, None, 0, None) == -1 and "null" in _err()
    assert fn(None, p[1], p[2], 1, 10, p[3], 1, p[4], None, p[5], 0, None, None, 0, None) == -1
    assert "not finalized" in _err()


def _visible(R=8, O=3, N=642, G=2, A=4, metric=0, k=5, HW=1024, null=None):
    p = [_fake() for _ in range(8)]
    if null is not None:
        p[null] = None
    rc = _lib().nope_score_topk_visible(p[0], p[1], R, O, N, CL, HW, p[2], p[3], G, A, p[4], metric, 0.2, k, p[5],
                                        p[6], p[7], None)
    return rc, _err()


def test_score_topk_visible_refusals():
    for null in range(6):                                   # query, emb, slots, row_off, visible, sim
        rc, msg = _visible(null=null)
        assert rc == -1 and "null" in msg, null
    for null in (6, 7):                                     # top-k outputs, with k > 0
        rc, msg = _visible(null=null)
        assert rc == -1 and "top-k" in msg
    for kw, word in (({"G": 0}, "G"), ({"G": 65536}, "G"), ({"R": 10, "A": 4}, "multiple of A"), ({"A": 0}, "A"),
                     ({"k": 65}, "k must"), ({"N": 3, "A": 1, "k": 4}, "k must"), ({"O": 65536}, "too many"),
                     ({"R": 4096, "A": 1, "HW": 2 ** 20}, "visible map"), ({"metric": 3}, "metric"),
                     ({"R": 0}, "bad arguments"), ({"HW": 0}, "bad arguments")):
        rc, msg = _visible(**kw)
        assert rc == -1 and word in msg, (kw, msg)


# ------------------------------------------------------------------ the Python layer, before any device work
def _model():
    from nope_b200.model import PoseConditional

    def sweep(*a, **kw):
        raise AssertionError("device work before the refusal")
    e = type("UNet", (), {})()
    e.channels, e.precision, e.device, e.sweep = CL, "fp16", torch.device("cpu"), sweep
    e.encoder = types.SimpleNamespace(precision="split", latent_dim=CL)
    return PoseConditional(e)


def test_python_refusals():
    from nope_b200.visibility import check_hidden
    m = _model()
    q, ref, rel = torch.zeros(2, 3, 256, 256), torch.zeros(2, 3, 256, 256), torch.zeros(2, 5, 6)
    for bad, word in ((torch.zeros(2, 256, 256), "uint8 or bool"), (torch.zeros(2, 128, 128, dtype=torch.uint8), "expected"),
                      (torch.zeros(3, 256, 256, dtype=torch.bool), "expected"), (np.zeros((2, 256, 256), np.uint8), "uint8")):
        for fn in (lambda: m.predict_pose(q, ref, rel, hidden=bad),
                   lambda: m.predict_pose_inplane(q, ref, rel, angles=4, hidden=bad),
                   lambda: m.retrieval_inplane(q, torch.zeros(2, 5, CL, 32, 32), angles=4, hidden=bad),
                   lambda: m.retrieval(q, torch.zeros(2, 5, CL, 32, 32), hidden=bad)):
            with pytest.raises(ValueError, match=word):
                fn()
    ok = torch.zeros(2, 256, 256, dtype=torch.uint8)
    m.dist = object()
    with pytest.raises(NotImplementedError, match="one device"):
        m.predict_pose(q, ref, rel, hidden=ok)
    with pytest.raises(NotImplementedError, match="does not shard"):
        m.predict_pose_inplane(q, ref, rel, angles=4, hidden=ok)
    with pytest.raises(NotImplementedError, match="one device"):
        m.retrieval_inplane(q, torch.zeros(2, 5, CL, 32, 32), angles=4, hidden=ok)
    with pytest.raises(NotImplementedError, match="one device"):
        m.retrieval(q, torch.zeros(2, 5, CL, 32, 32), hidden=ok)
    # the multi-query form: hidden follows the query's leading shape
    with pytest.raises(ValueError, match=r"\(2, 3, 256, 256\)"):
        check_hidden(ok, (2, 3), "predict_pose")


def test_occluded_search_needs_occluders():
    m = _model()
    frames, masks, K = torch.zeros(1, 8, 8, 3, dtype=torch.uint8), torch.zeros(2, 8, 8, dtype=torch.uint8), torch.eye(3)
    for fn in (lambda: m.predict_pose_frames(frames, masks, K, [4, 9], occluded_search=True),
               lambda: m.track_pose_frames(frames, masks, K, [4, 9], torch.zeros(2, 1, 3, 3), _refiner(),
                                           occluded_search=True)):
        with pytest.raises(ValueError, match="needs occluders"):
            fn()
    m.dist = object()
    with pytest.raises(NotImplementedError, match="one device"):
        m.predict_pose_frames(frames, masks, K, [4, 9], occluders="detections", occluded_search=True)


def _refiner():
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations
    return InplaneRefiner(torch.from_numpy(icosphere_object_rotations(0)), 4, 1)


def test_roll_sample_is_the_inplane_oracles():
    """oracle/inplane_oracle.rotate keeps its sample inside the rotation; the visibility oracle restates it.  The
    bilinear image rebuilt from roll_sample's taps and fractions, in rotate's lerp order, is rotate's output bit for
    bit, so the two samples cannot drift apart unnoticed."""
    from oracle import inplane_oracle
    g = torch.Generator().manual_seed(2)
    img = torch.rand(1, 3, 256, 256, generator=g) * 2 - 1
    t = torch.tensor([0.3, 1.1, 2.9, 4.4])
    cs = torch.cat([torch.stack([t.cos(), t.sin()], 1), torch.tensor([[0.0, 1.0], [-1.0, 0.0]])]).float()
    ref = inplane_oracle.rotate(img, cs)[0]                                   # [A, 3, 256, 256]
    for a in range(cs.shape[0]):
        ix, iy, fx, fy = (torch.from_numpy(x) for x in vo.roll_sample(cs[a, 0].item(), cs[a, 1].item(), 256))

        def tap(yy, xx):
            inside = (yy >= 0) & (yy < 256) & (xx >= 0) & (xx < 256)
            return torch.where(inside, img[0][:, yy.clamp(0, 255), xx.clamp(0, 255)], torch.tensor(-1.0))
        v00, v01, v10, v11 = tap(iy, ix), tap(iy, ix + 1), tap(iy + 1, ix), tap(iy + 1, ix + 1)
        top = v00 + fx * (v01 - v00)
        bot = v10 + fx * (v11 - v10)
        assert torch.equal(top + fy * (bot - top), ref[a]), a
