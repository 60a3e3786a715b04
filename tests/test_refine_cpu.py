"""CPU: the off-grid pose refinement without a device -- the lattice stencil and the grid spacing it starts from,
the torch oracle's propose / select conventions (and a whole refinement of a smooth synthetic score with it), the
ABI's refusals, and the Python argument errors."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from oracle import refine_oracle as orc


def _angle(R):
    return np.arccos(np.clip((np.trace(R, axis1=-2, axis2=-1) - 1.0) / 2.0, -1.0, 1.0))


# ------------------------------------------------------------------ stencil and spacing
@pytest.mark.parametrize("theta", [0.07, 0.003])
def test_stencil_rotations(theta):
    from nope_b200.refine import stencil
    L = stencil(theta)
    assert L.shape == (27, 3, 3)
    assert np.array_equal(L[0], np.eye(3))                                        # identity first, exactly
    assert np.allclose(L @ L.transpose(0, 2, 1), np.eye(3), atol=1e-14)
    assert np.allclose(np.linalg.det(L), 1.0, atol=1e-14)
    ang = _angle(L[1:]) / theta
    assert np.allclose(np.sort(ang), np.sort([1.0] * 6 + [math.sqrt(2)] * 12 + [math.sqrt(3)] * 8), atol=1e-6)
    # slots 1..26: the rotation vectors (i, j, l) in lexicographic order, (0, 0, 0) left out
    offs = [(i, j, l) for i in (-1, 0, 1) for j in (-1, 0, 1) for l in (-1, 0, 1) if (i, j, l) != (0, 0, 0)]
    for Lj, v in zip(L[1:], offs):
        w = np.array([Lj[2, 1] - Lj[1, 2], Lj[0, 2] - Lj[2, 0], Lj[1, 0] - Lj[0, 1]]) / 2.0   # sin(phi) * axis
        phi = theta * np.linalg.norm(v)
        assert np.allclose(w, np.sin(phi) * np.asarray(v) / np.linalg.norm(v), atol=1e-14)
    assert np.allclose(L, orc.stencil(theta).numpy(), atol=1e-15)


@pytest.mark.parametrize("level,spacing_deg", [(1, 16.4), (2, 8.3), (3, 4.2)])
def test_theta0_is_half_the_median_nearest_neighbour_angle(level, spacing_deg):
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.refine import PoseRefiner
    R = icosphere_object_rotations(level)
    A = R.reshape(len(R), 9)
    t = A @ A.T
    np.fill_diagonal(t, -np.inf)
    direct = 0.5 * np.median(np.arccos(np.clip((t.max(axis=1) - 1.0) / 2.0, -1.0, 1.0)))
    ref = PoseRefiner(R, steps=3)
    assert ref.num_poses == len(R)
    assert abs(ref.theta0 - direct) < 1e-9
    assert abs(math.degrees(2 * ref.theta0) - spacing_deg) < 0.1
    assert ref.thetas == (ref.theta0, ref.theta0 / 2, ref.theta0 / 4)
    assert ref.stencils.shape == (3, 27, 9) and ref.stencils.dtype == torch.float32
    for s, th in enumerate(ref.thetas):
        assert torch.equal(ref.stencils[s], torch.from_numpy(orc.stencil(th).numpy().astype(np.float32)).view(27, 9))
        assert ref.thresholds[s] == float(np.float32(1 + 2 * math.cos(th / 2)))
    assert ref.hypotheses(4) == len(R) + 3 * 4 * 27


# ------------------------------------------------------------------ oracle conventions
def _rot(axis, angle):
    from nope_b200.refine import axis_angle_matrix
    return torch.from_numpy(axis_angle_matrix(np.asarray(axis, dtype=np.float64) * angle)).float()


def test_oracle_propose_slots_and_padding():
    from nope_b200.refine import stencil
    g = torch.Generator().manual_seed(0)
    grid = torch.stack([_rot(torch.randn(3, generator=g).tolist(), 0.5 + 0.1 * n) for n in range(5)])
    poses = grid[None, :, :2].reshape(1, 5, 6).expand(2, 5, 6).contiguous()          # B = 2 references
    L = torch.from_numpy(stencil(0.05).astype(np.float32)).view(27, 9)
    D = torch.stack([_rot([0, 0, 1], 0.01), _rot([1, 0, 0], -0.02), torch.eye(3)]).view(1, 3, 9).repeat(4, 1, 1)
    seed = torch.tensor([[3, 9, 1], [-1, 2, 2], [5, -2, 7], [0, 4, 1]], dtype=torch.int32)   # R = B * Q, Q = 2
    out = orc.propose(D, seed, poses, L, Q=2)
    M = 81
    assert out["D"].shape == (4, M, 9) and out["poses"].shape == (4, M, 6)
    assert out["seed"][0].tolist() == [3] * 27 + [-1] * 27 + [1] * 27
    assert torch.equal(out["D"][0, 0], D[0, 0])                                   # slot 0: identity * D
    assert torch.equal(out["rel"][0, 27:54], out["rel"][0, :1].expand(27, 9))     # padding: the first candidate
    assert torch.equal(out["D"][1, :27], out["D"][1, 27:28].expand(27, 9))        # first valid centre is centre 1
    assert (out["seed"][2] == -1).all()                                           # no valid centre: I at seed 0
    assert torch.equal(out["D"][2], torch.eye(3).reshape(1, 9).expand(M, 9))
    assert torch.equal(out["rel"][2, 0].view(3, 3), orc.mat3_mul(torch.eye(3), orc.seed_rotation(poses[1, 0])))
    rel = out["rel"][3, 27 * 1 + 5].double().view(3, 3)                           # (L_5 D_1) S_4, reference 1
    want = L[5].double().view(3, 3) @ D[3, 1].double().view(3, 3) @ grid[4].double()
    assert torch.allclose(rel, want, atol=1e-6)
    assert torch.equal(out["poses"], out["rel"][..., :6])


def _cands(rels, seeds):
    rel = torch.stack([r.reshape(9) for r in rels])[None]
    return {"D": rel.clone(), "rel": rel, "seed": torch.tensor([seeds], dtype=torch.int32)}


def test_oracle_select_suppresses_duplicates_ties_to_lowest_slot_and_skips_padding():
    a, b, c = _rot([0, 0, 1], 0.0), _rot([0, 0, 1], 0.012), _rot([0, 1, 0], 0.3)
    thr = float(np.float32(1 + 2 * math.cos(0.02 / 2)))                           # theta = 0.02: b is 0.012 from a
    cand = _cands([a, a, b, c, c, a], [1, 2, 1, 3, 3, -1])
    sim = torch.tensor([[5.0, 5.0, 4.0, 7.0, 7.0, 9.0]])
    out = orc.select(sim, cand, thr, 4)
    # padding (9.0) is never chosen; slot 3 wins its tie with slot 4, which it then suppresses; slot 0 likewise
    # wins against and suppresses slot 1; b lies beyond theta / 2 of a and stays; then nothing is left
    assert out["seed"].tolist() == [[3, 1, 1, -1]]
    assert out["score"][0, :3].tolist() == [7.0, 5.0, 4.0] and out["score"][0, 3] == float("-inf")
    assert torch.equal(out["rel"][0, 0], c.reshape(9)) and torch.equal(out["rel"][0, 2], b.reshape(9))
    assert (out["D"][0, 3] == 0).all()
    # theta = 0.03: b lies within theta / 2 = 0.015 of a and goes too
    thr = float(np.float32(1 + 2 * math.cos(0.03 / 2)))
    out = orc.select(sim, cand, thr, 4)
    assert out["seed"].tolist() == [[3, 1, -1, -1]]


def test_oracle_refinement_of_a_smooth_score_goes_below_the_grid():
    """the refinement restated entirely in the oracle, on a smooth synthetic score (minus the squared geodesic
    distance to a hidden off-grid target): the best score never decreases and the result lies far below the grid's
    spacing"""
    from nope_b200.poses import icosphere_object_rotations, matrix_to_rotation_6d
    from nope_b200.refine import PoseRefiner
    R = icosphere_object_rotations(1)
    ref = PoseRefiner(R, steps=5)
    poses = matrix_to_rotation_6d(torch.from_numpy(R).float())[None]
    target = (_rot([0.3, -0.5, 0.8], 0.09).double() @ torch.from_numpy(R[17])).reshape(9)

    def score(rel):
        t = (rel.double() * target).sum(-1)
        return (-torch.arccos(((t - 1) / 2).clamp(-1, 1)) ** 2).float()

    grid_scores = score(orc.mat3_mul(torch.eye(3), orc.seed_rotation(poses[0])).reshape(-1, 9))
    keep = 3
    seed = torch.sort(-grid_scores, stable=True).indices[:keep].to(torch.int32)[None]
    cur = {"D": torch.eye(3).reshape(1, 1, 9).expand(1, keep, 9).contiguous(), "seed": seed}
    best = [float(grid_scores.max())]
    for s in range(ref.steps):
        cand = orc.propose(cur["D"], cur["seed"], poses, ref.stencils[s], 1)
        sim = score(cand["rel"])
        cur = orc.select(sim, cand, ref.thresholds[s], keep)
        best.append(float(cur["score"][0, 0]))
    assert all(b1 >= b0 for b0, b1 in zip(best, best[1:])), best
    grid_err = math.sqrt(-best[0])
    final_err = math.sqrt(-best[-1])
    assert final_err < ref.thetas[-1] < grid_err, (grid_err, final_err)


# ------------------------------------------------------------------ ABI
@pytest.mark.parametrize("R,keep,B,Q,needle", [(2, 0, 2, 1, "keep"), (2, 65, 2, 1, "keep"), (3, 2, 2, 1, "R")])
def test_propose_rejects_bad_sizes(R, keep, B, Q, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    p = C.c_void_p(256)
    assert lib.nope_pose_refine_propose(p, p, R, keep, p, B, Q, 10, p, p, p, p, p, None) != 0
    assert needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("M,k,needle", [(27, 0, "k"), (1728, 65, "k"), (27, 28, "k"), (1729, 5, "M")])
def test_select_rejects_bad_sizes(M, k, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    p = C.c_void_p(256)
    assert lib.nope_pose_refine_select(p, p, p, p, 2, M, k, 2.9, p, p, p, None, None) != 0
    assert needle in lib.nope_last_error().decode()


# ------------------------------------------------------------------ Python argument errors
class _NoDevice:
    """an engine that fails the test if any work reaches it"""
    device = torch.device("cpu")

    def sweep(self, *a, **kw):
        raise AssertionError("device work before the argument check")


def test_python_argument_errors_without_a_device():
    from nope_b200.ldm import UNetModelPose
    from nope_b200.model import PoseConditional
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.refine import PoseRefiner, refine
    R = icosphere_object_rotations(0)
    ref = PoseRefiner(R, steps=2)
    rel = torch.zeros(1, 42, 6)
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    ldm = UNetModelPose(device="cpu")
    img, lat = torch.zeros(1, 3, 256, 256), torch.zeros(1, 4, 32, 32)
    with pytest.raises(ValueError):
        PoseRefiner(R[:1])
    with pytest.raises(ValueError):
        PoseRefiner(R, steps=0)
    bad = [dict(keep=0), dict(keep=65), dict(k=0), dict(k=65), dict(keep=1, k=28),        # ranges, k > keep * 27
           dict(all_relativeR=torch.zeros(1, 41, 6)),                                     # grid size != refiner
           dict(all_relativeR=torch.zeros(2, 42, 6)),                                     # references != batch
           dict(all_relativeR=torch.zeros(1, 42, 9)),
           dict(refiner=object())]
    for kw in bad:
        kw = {"all_relativeR": rel, "refiner": ref, **kw}
        with pytest.raises(ValueError):
            model.predict_pose_refined(img, img, **kw)
        with pytest.raises(ValueError):
            ldm.predict_pose_refined(lat, lat, **kw)
    with pytest.raises(ValueError):                                                       # keep > N
        model.predict_pose_refined(img, img, torch.zeros(1, 2, 6), PoseRefiner(R[:2]), k=5, keep=3)
    eng, feat = _NoDevice(), torch.zeros(2, 8, 32, 32)
    seeds = torch.zeros(2, 4, dtype=torch.int64)
    rel2 = torch.zeros(2, 42, 6)
    for args, kw in [((rel2, seeds[:, :0]), {}), ((rel2, torch.zeros(2, 65, dtype=torch.int64)), {}),
                     ((rel2, seeds), dict(k=109)), ((rel2[:1], seeds), {}), ((rel2, seeds[:1]), {}),
                     ((rel2, seeds[:, None]), {})]:
        with pytest.raises(ValueError):
            refine(eng, feat, feat, *args, ref, **kw)


def test_sharded_model_is_refused():
    from nope_b200.model import PoseConditional
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.refine import PoseRefiner
    R = icosphere_object_rotations(0)
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    model.dist = object()
    img = torch.zeros(1, 3, 256, 256)
    with pytest.raises(NotImplementedError, match="shard"):
        model.predict_pose_refined(img, img, torch.zeros(1, 42, 6), PoseRefiner(R))
