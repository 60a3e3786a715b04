"""CPU: the joint roll and viewpoint refinement without a device -- the xy stencil and the step schedule, the torch
oracle's propose / select conventions (and a whole refinement of a smooth synthetic score with it), the ABI's
refusals, and the Python argument errors."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from oracle import inplane_refine_oracle as orc
from oracle import refine_oracle


def _angle(R):
    return np.arccos(np.clip((np.trace(R, axis1=-2, axis2=-1) - 1.0) / 2.0, -1.0, 1.0))


# ------------------------------------------------------------------ stencil and schedule
@pytest.mark.parametrize("theta", [0.07, 0.003])
def test_xy_stencil(theta):
    from nope_b200.inplane_refine import xy_stencil
    L = xy_stencil(theta)
    assert L.shape == (9, 3, 3)
    assert np.array_equal(L[0], np.eye(3))                                        # identity first, exactly
    assert np.allclose(L @ L.transpose(0, 2, 1), np.eye(3), atol=1e-14)
    offs = [(i, j) for i in (-1, 0, 1) for j in (-1, 0, 1) if (i, j) != (0, 0)]   # lexicographic
    for Lj, (i, j) in zip(L[1:], offs):
        w = np.array([Lj[2, 1] - Lj[1, 2], Lj[0, 2] - Lj[2, 0], Lj[1, 0] - Lj[0, 1]]) / 2.0   # sin(phi) * axis
        phi = theta * math.hypot(i, j)
        assert abs(_angle(Lj) - phi) < 1e-9                                       # angle theta * |(i, j)|
        assert w[2] == 0.0                                                        # no z component
        assert np.allclose(w, np.sin(phi) * np.array([i, j, 0.0]) / math.hypot(i, j), atol=1e-14)
    assert np.allclose(L, orc.xy_stencil(theta).numpy(), atol=1e-15)


@pytest.mark.parametrize("level", [1, 2, 3])
@pytest.mark.parametrize("A", [12, 36])
def test_schedule_matches_pose_refiner_and_half_bins(level, A):
    from nope_b200.inplane_refine import InplaneRefiner, xy_stencil
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.refine import PoseRefiner
    R = icosphere_object_rotations(level)
    steps = 4
    ir, pr = InplaneRefiner(R, angles=A, steps=steps), PoseRefiner(R, steps=steps)
    assert ir.thetas == pr.thetas and ir.num_poses == len(R) and ir.angles == A
    assert np.allclose(ir.phis, [math.radians(180.0 / A) * 2.0 ** -s for s in range(steps)], rtol=1e-15, atol=0)
    assert ir.stencils.shape == (steps, 9, 9) and ir.stencils.dtype == torch.float32
    for s in range(steps):
        assert torch.equal(ir.stencils[s], torch.from_numpy(xy_stencil(ir.thetas[s]).astype(np.float32)).view(9, 9))
        assert ir.rolls[s] == (float(np.float32(math.cos(ir.phis[s]))), float(np.float32(math.sin(ir.phis[s]))))
        psi = min(ir.thetas[s], ir.phis[s])
        assert ir.thresholds[s] == float(np.float32(1 + 2 * math.cos(psi / 2)))
    assert ir.hypotheses(2) == steps * 2 * 9 and ir.crops(2) == steps * 2 * 2


# ------------------------------------------------------------------ oracle conventions
def _rot(axis, angle):
    from nope_b200.refine import axis_angle_matrix
    return torch.from_numpy(axis_angle_matrix(np.asarray(axis, dtype=np.float64) * angle)).float()


def _cs(deg):
    return torch.tensor([math.cos(math.radians(deg)), math.sin(math.radians(deg))], dtype=torch.float32)


def test_oracle_propose_slots_and_padding():
    from nope_b200.inplane_refine import xy_stencil
    g = torch.Generator().manual_seed(0)
    grid = torch.stack([_rot(torch.randn(3, generator=g).tolist(), 0.5 + 0.1 * n) for n in range(5)])
    poses = grid[None, :, :2].reshape(1, 5, 6).expand(2, 5, 6).contiguous()          # B = 2 references
    L = torch.from_numpy(xy_stencil(0.05).astype(np.float32)).view(9, 9)
    D = torch.stack([_rot([0, 0, 1], 0.01), _rot([1, 0, 0], -0.02), torch.eye(3)]).view(1, 3, 9).repeat(4, 1, 1)
    seed = torch.tensor([[3, 9, 1], [-1, 2, 2], [5, -2, 7], [0, 4, 1]], dtype=torch.int32)
    cs = torch.stack([_cs(10), _cs(-40), _cs(170)]).view(1, 3, 2).repeat(4, 1, 1)
    roll = (float(np.float32(math.cos(0.1))), float(np.float32(math.sin(0.1))))
    out = orc.propose(D, seed, cs, poses, L, roll, Q=2)
    assert out["D"].shape == (4, 27, 9) and out["cossin"].shape == (4, 9, 2)
    assert out["seed"][0].tolist() == [3] * 9 + [-1] * 9 + [1] * 9
    assert torch.equal(out["cossin"][0, 0], cs[0, 0])                             # l = 0: rho bit for bit
    c, s = float(cs[0, 0, 0]), float(cs[0, 0, 1])
    want = [c * roll[0] - s * roll[1], s * roll[0] + c * roll[1]]
    assert torch.allclose(out["cossin"][0, 1].double(), torch.tensor(want, dtype=torch.float64), atol=1e-7)
    ang = [math.degrees(math.atan2(float(v[1]), float(v[0]))) for v in out["cossin"][0, :3]]
    assert np.allclose(ang, [10, 10 + math.degrees(0.1), 10 - math.degrees(0.1)], atol=1e-4)
    assert torch.equal(out["cossin"][0, 3:6], cs[0, 0].expand(3, 2))              # padding centre: centre 0's rho
    assert torch.equal(out["cossin"][1, 0:3], cs[1, 1].expand(3, 2))              # first valid centre is centre 1
    assert (out["seed"][2] == -1).all() and torch.equal(out["cossin"][2], torch.tensor([1.0, 0.0]).expand(9, 2))
    rel = out["rel"][3, 9 * 1 + 5].double().view(3, 3)                            # (L_5 D_1) S_4, reference 1
    assert torch.allclose(rel, L[5].double().view(3, 3) @ D[3, 1].double().view(3, 3) @ grid[4].double(), atol=1e-6)
    assert torch.equal(out["poses"], out["rel"][..., :6])


def _cand(rels, seeds, rolls):
    """keep = 1: 9 pose slots (rels padded with copies of the first), 3 angle slots"""
    rel = torch.stack([r.reshape(9) for r in rels] + [rels[0].reshape(9)] * (9 - len(rels)))[None]
    seed = torch.tensor([list(seeds) + [seeds[0]] * (9 - len(seeds))], dtype=torch.int32)
    return {"D": rel.clone(), "rel": rel, "seed": seed, "cossin": torch.stack(rolls)[None]}


def test_oracle_select_ties_padding_duplicates_and_cross_centre_pairs():
    a, b = _rot([0, 0, 1], 0.0), _rot([0, 1, 0], 0.3)
    thr = float(np.float32(1 + 2 * math.cos(0.02 / 2)))
    cand = _cand([a, b, b, a], [1, 2, -1, 4], [_cs(0), _cs(40), _cs(0)])
    sim = torch.full((1, 3, 9), -10.0)
    sim[0, 0, 2] = 99.0                                                          # padding pose slot: never chosen
    sim[0, 0, 1] = sim[0, 2, 1] = 7.0                                            # a tie of exact duplicates:
    sim[0, 1, 3] = 6.0                                                           # (a0, p1) wins, (a2, p1) dropped
    out = orc.select(sim, cand, thr, 3)
    assert out["aslot"][0].tolist()[:2] == [0, 1] and out["seed"][0].tolist()[:2] == [2, 4]
    assert out["score"][0, :2].tolist() == [7.0, 6.0]
    assert torch.equal(out["cossin"][0, 1], _cs(40)) and torch.equal(out["rel"][0, 1], a.reshape(9))
    # the third: the lowest remaining pair, (a0, p0), 0.3 rad from the first and 40 degrees from the second
    assert out["score"][0, 2] == -10.0 and out["aslot"][0, 2] == 0 and out["seed"][0, 2] == 1
    E = orc.pair_rotations(cand)[0]
    assert torch.equal(E[1], E[19]) and torch.equal(E[0], a.reshape(9))             # the dropped exact duplicate
    # angle slots whose centre is padding (seed -1) are never chosen either
    cand2 = _cand([a, b], [-1, 2], [_cs(0), _cs(10), _cs(20)])
    out2 = orc.select(torch.zeros(1, 3, 9), cand2, thr, 2)
    assert out2["seed"].tolist() == [[-1, -1]] and torch.isneginf(out2["score"]).all()
    assert (out2["aslot"] == -1).all() and (out2["cossin"] == 0).all()


def test_oracle_select_cross_centre_pairs_are_selectable():
    """keep = 2: the best pair joins centre 1's roll with centre 0's pose"""
    a, b = _rot([1, 0, 0], 0.2), _rot([0, 1, 0], -0.4)
    rel = torch.cat([a.reshape(1, 9).expand(9, 9), b.reshape(1, 9).expand(9, 9)])[None].contiguous()
    seed = torch.tensor([[3] * 9 + [5] * 9], dtype=torch.int32)
    cs = torch.stack([_cs(0), _cs(5), _cs(-5), _cs(90), _cs(95), _cs(85)])[None]
    cand = {"D": rel.clone(), "rel": rel, "seed": seed, "cossin": cs}
    sim = torch.zeros(1, 6, 18)
    sim[0, 3, 0] = 1.0                                                           # angle slot 3 (centre 1), pose 0
    out = orc.select(sim, cand, float(np.float32(1 + 2 * math.cos(0.01))), 1)
    assert out["aslot"].tolist() == [[3]] and out["seed"].tolist() == [[3]]
    assert torch.equal(out["cossin"][0, 0], _cs(90)) and torch.equal(out["rel"][0, 0], a.reshape(9))


def test_oracle_refinement_of_a_smooth_score_converges():
    """the whole refinement restated in the oracle on a smooth score over (roll, viewpoint): minus the squared
    geodesic distance of Rz(rho) D S to a hidden target off the bins and off the grid.  The best score never
    decreases, and the result lies far below the bin and grid spacing."""
    from nope_b200.inplane import inplane_rotations, inplane_table
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations, matrix_to_rotation_6d
    Rg = icosphere_object_rotations(1)
    A = 12
    ref = InplaneRefiner(Rg, angles=A, steps=6)
    poses = matrix_to_rotation_6d(torch.from_numpy(Rg).float())[None]
    beta = math.radians(13.7)
    Rzb = torch.tensor([[math.cos(beta), -math.sin(beta), 0], [math.sin(beta), math.cos(beta), 0], [0, 0, 1]],
                       dtype=torch.float64)
    target = (Rzb @ _rot([0.6, -0.8, 0.0], 0.08).double() @ torch.from_numpy(Rg[17])).reshape(9)

    def score(E):
        t = (E.double() * target).sum(-1)
        return (-torch.arccos(((t - 1) / 2).clamp(-1, 1)) ** 2).float()

    S = refine_oracle.seed_rotation(poses[0]).double()                           # [N, 3, 3]
    grid = score((inplane_rotations(A)[:, None] @ S[None]).reshape(A, -1, 9))     # [A, N]
    keep = 2
    flat = torch.sort(-grid.reshape(-1), stable=True).indices[:keep]
    n, a = flat % len(Rg), flat // len(Rg)
    cur = {"D": torch.eye(3).reshape(1, 1, 9).expand(1, keep, 9).contiguous(),
           "seed": n.to(torch.int32)[None], "cossin": inplane_table(A)[a][None]}
    best = [float(grid.max())]
    for s in range(ref.steps):
        cand = orc.propose(cur["D"], cur["seed"], cur["cossin"], poses, ref.stencils[s], ref.rolls[s], 1)
        sim = score(orc.pair_rotations(cand)).view(1, keep * 3, keep * 9)
        cur = orc.select(sim, cand, ref.thresholds[s], keep)
        best.append(float(cur["score"][0, 0]))
    assert all(b1 >= b0 for b0, b1 in zip(best, best[1:])), best
    start, final = math.sqrt(-best[0]), math.sqrt(-best[-1])
    assert final < 0.1 * start and final < min(ref.thetas[-1], ref.phis[-1]), (start, final)


# ------------------------------------------------------------------ ABI
P = C.c_void_p(256)     # never dereferenced: every case below is refused before any CUDA call


@pytest.mark.parametrize("args,needle", [
    ((None, 1, 8, 8, P, P, 1, P), "null"), ((P, 1, 8, 8, None, P, 1, P), "null"),
    ((P, 0, 8, 8, P, P, 1, P), "B"), ((P, 1, 0, 8, P, P, 1, P), "H"), ((P, 1, 8, 8, P, P, 0, P), "P")])
def test_rotate_pairs_refusals(args, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_inplane_rotate_pairs(*args, None) != 0
    assert needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("args,needle", [((None, P, 1, P, P, 1, P), "encoder"), ((P, None, 1, P, P, 1, P), "null"),
                                         ((P, P, 1, None, P, 1, P), "null"), ((P, P, 1, P, P, 0, P), "P"),
                                         ((P, P, 0, P, P, 1, P), "B")])
def test_encode_rotated_refusals(args, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_encoder_encode_rotated(*args, None) != 0
    assert needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("R,keep,B,Q,null,needle", [(2, 0, 2, 1, False, "keep"), (2, 17, 2, 1, False, "keep"),
                                                    (3, 2, 2, 1, False, "R"), (2, 2, 2, 1, True, "null")])
def test_propose_refusals(R, keep, B, Q, null, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_pose_refine_inplane_propose(P, P, None if null else P, R, keep, P, B, Q, 10, P, 1.0, 0.0,
                                                P, P, P, P, P, None) != 0
    assert needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("keep,k,null,needle", [(2, 0, False, "k"), (16, 65, False, "k"), (1, 28, False, "k"),
                                                (0, 1, False, "keep"), (17, 1, False, "keep"), (2, 5, True, "null")])
def test_select_refusals(keep, k, null, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_pose_refine_inplane_select(P, P, P, P, P, 2, keep, k, 2.9, P, P, P, None if null else P, P,
                                               None, None) != 0
    assert needle in lib.nope_last_error().decode()


def test_select_accepts_the_largest_k():
    """k = 27 * keep^2 at keep = 1 passes the size checks (refused here only for R = 0, still before any launch)"""
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_pose_refine_inplane_select(P, P, P, P, P, 0, 1, 27, 2.9, P, P, P, P, P, None, None) != 0
    assert "bad arguments" in lib.nope_last_error().decode()


# ------------------------------------------------------------------ Python argument errors
class _NoDevice:
    """an engine that fails the test if any work reaches it"""
    device = torch.device("cpu")

    def sweep(self, *a, **kw):
        raise AssertionError("device work before the argument check")


def test_python_argument_errors_without_a_device():
    from nope_b200.inplane_refine import InplaneRefiner, refine_inplane
    from nope_b200.model import PoseConditional
    from nope_b200.poses import icosphere_object_rotations
    R = icosphere_object_rotations(0)
    ref = InplaneRefiner(R, angles=12, steps=2)
    rel = torch.zeros(1, 42, 6)
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    img = torch.zeros(1, 3, 256, 256)
    for kw in (dict(angles=0), dict(angles=361), dict(steps=0), dict(steps=1.5)):
        with pytest.raises(ValueError):
            InplaneRefiner(R, **kw)
    with pytest.raises(ValueError):
        InplaneRefiner(R[:1])
    bad = [dict(keep=0), dict(keep=17), dict(k=0), dict(k=65), dict(keep=1, k=28), dict(keep=1.0),
           dict(all_relativeR=torch.zeros(1, 41, 6)), dict(all_relativeR=torch.zeros(2, 42, 6)),
           dict(all_relativeR=torch.zeros(1, 42, 9)), dict(refiner=object())]
    for kw in bad:
        kw = {"all_relativeR": rel, "refiner": ref, **kw}
        with pytest.raises(ValueError):
            model.predict_pose_inplane_refined(img, img, **kw)
    with pytest.raises(ValueError):                                                # keep > A * N
        model.predict_pose_inplane_refined(img, img, torch.zeros(1, 2, 6), InplaneRefiner(R[:2], angles=1),
                                           k=5, keep=3)
    with pytest.raises(ValueError):                                                # query does not fit
        model.predict_pose_inplane_refined(torch.zeros(2, 3, 3, 256, 256), img, rel, ref)
    eng, feat = _NoDevice(), torch.zeros(2, 8, 32, 32)
    imgs, rel2 = torch.zeros(2, 3, 256, 256), torch.zeros(2, 42, 6)
    s2 = torch.zeros(2, 2, dtype=torch.int64)
    lat = torch.zeros(2, 2, 8, 32, 32)
    for args, kw in [((imgs, rel2, (s2, s2), lat), dict(k=109)),                   # k > 27 keep^2
                     ((imgs, rel2, (s2[:, :0], s2[:, :0]), lat[:, :0]), {}),       # keep = 0
                     ((imgs, rel2[:1], (s2, s2), lat), {}),                        # references
                     ((imgs[:1], rel2, (s2, s2), lat), {}),                        # images
                     ((imgs, rel2, (s2, s2[:, :1]), lat), {}),                     # seed shapes
                     ((imgs, rel2, (s2, s2), lat[:, :1]), {})]:                    # latent shape
        with pytest.raises(ValueError):
            refine_inplane(eng, None, feat, *args, ref, **kw)


def test_sharded_model_is_refused():
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.model import PoseConditional
    from nope_b200.poses import icosphere_object_rotations
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    model.dist = object()
    img = torch.zeros(1, 3, 256, 256)
    with pytest.raises(NotImplementedError, match="shard"):
        model.predict_pose_inplane_refined(img, img, torch.zeros(1, 42, 6),
                                           InplaneRefiner(icosphere_object_rotations(0)))
