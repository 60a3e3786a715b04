"""GPU: pose tracking (DESIGN.md section 26).  track_seed_kernel against the numpy oracle bit for bit; refine_inplane
with explicit centres against the tuple form; track_inplane's scores against separate sweeps and its seeds;
track_pose_frames against the chain of its stages, with a bank and with references, and its host synchronisations;
PoseTracker's searched, tracked, lost, new and dropped rows; and roll tracking over 48 frames through a stub engine
whose templates do not depend on the pose.  The weights are seeded: nothing here says how well a trained model
tracks."""
import numpy as np
import pytest
import torch

import track_oracle as to
from _scenes import H, K3, W, make_mesh, pose, rot, with_objects
from _util import count_host_syncs, same_bits

pytestmark = pytest.mark.gpu

A, KEEP, K = 6, 2, 3


def _seeds_raw(Rc, T):
    """nope_track_seeds on device copies of Rc [H, 3, 3] and T [N, 3, 3] (float64 numpy)"""
    from nope_b200 import _lib
    rc, t = torch.from_numpy(np.ascontiguousarray(Rc)).cuda(), torch.from_numpy(np.ascontiguousarray(T)).cuda()
    n = rc.shape[0]
    D = torch.empty(n, 3, 3, device="cuda")
    seed = torch.empty(n, device="cuda", dtype=torch.int32)
    cs = torch.empty(n, 2, device="cuda")
    _lib.check(_lib.load().nope_track_seeds(_lib.ptr(rc), n, _lib.ptr(t), t.shape[0], _lib.ptr(D), _lib.ptr(seed),
                                            _lib.ptr(cs), None))
    return D.cpu().numpy(), seed.cpu().numpy(), cs.cpu().numpy()


# ------------------------------------------------------------------ the seed kernel = the oracle
@pytest.mark.parametrize("level", [0, 2, 3])
@pytest.mark.parametrize("Hn", [1, 7, 96])
def test_seed_kernel_equals_the_oracle(level, Hn):
    """priors between grid poses, on grid poses (rolled), NaN / inf priors; a grid with duplicated rows (exact ties)
    and a NaN row"""
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.track import seed_centres
    grid = icosphere_object_rotations(level)
    assert len(grid) == {0: 42, 2: 642, 3: 2562}[level]
    rng = np.random.default_rng(100 * level + Hn)
    Rc = to.random_rotations(Hn, rng)
    if Hn > 1:
        on = rng.integers(0, len(grid), Hn // 2)
        Rc[1:1 + len(on)] = np.stack([to.rz(b) @ grid[i] for b, i in zip(rng.uniform(-180, 180, len(on)), on)])
        Rc[-1, 1, 2] = np.nan
    if Hn > 2:
        Rc[-2, 0, 0] = -np.inf
    want = to.track_seeds(Rc, grid)
    got = _seeds_raw(Rc, grid)
    for g, w in zip(got, want):
        assert same_bits(g, w)
    ref = InplaneRefiner(grid, angles=36, steps=1)
    cen = seed_centres(torch.from_numpy(Rc).cuda()[None], ref)
    assert cen["D"].shape == (1, Hn, 3, 3) and cen["seed"].shape == (1, Hn) and cen["cossin"].shape == (1, Hn, 2)
    for name, w in zip(("D", "seed", "cossin"), want):
        assert same_bits(cen[name][0].cpu().numpy(), w), name
    # float32 priors are widened exactly
    cen32 = seed_centres(torch.from_numpy(Rc).float().cuda(), ref)
    for name, w in zip(("D", "seed", "cossin"), to.track_seeds(Rc.astype(np.float32).astype(np.float64), grid)):
        assert same_bits(cen32[name].cpu().numpy(), w), name
    # ties and a NaN grid row
    T = grid.copy()
    T[-3:] = T[:3]
    T[5] = np.nan
    Rt = np.concatenate([Rc, np.stack([to.rz(11.0) @ grid[1], to.rz(-3.0) @ grid[5], grid[2]])])
    want = to.track_seeds(Rt, T)
    assert want[1][-3] == 1 and want[1][-2] != 5 and want[1][-1] == 2
    for g, w in zip(_seeds_raw(Rt, T), want):
        assert same_bits(g, w)


# ------------------------------------------------------------------ refine_inplane with centres
@pytest.fixture(scope="module")
def grids():
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    R2 = icosphere_object_rotations(2)
    return {"R": R2, "rel": synthetic_pose_batch(642, 3)[0].cuda(), "ref": InplaneRefiner(R2, angles=36, steps=2)}


@pytest.fixture(scope="module")
def scene():
    from oracle import inputs
    g = torch.Generator().manual_seed(31)
    q = (torch.rand(3, 3, 256, 256, generator=g) * 2 - 1).cuda()
    _, r = inputs.make_images(seed=11, batch=3)
    return {"q": q, "r": r.cuda()}


def test_centres_equal_the_tuple_form(gpu_model, grids, scene):
    from nope_b200.inplane_refine import refine_inplane
    from nope_b200.model import topk
    u, ref, rel = gpu_model.u_net, grids["ref"], grids["rel"]
    enc = u.encoder
    u.set_metric("l2")
    rf = enc.encode_image(scene["r"])
    qf = enc.encode_image_inplane(scene["q"], ref.angles)
    sim = u.sweep(rf, rel, query_feat=qf, want_emb=False, want_sim=True)["sim"]
    _, flat = topk(sim.view(3, -1), KEEP)
    n, a = flat % 642, flat // 642
    lat = qf[torch.arange(3, device=qf.device)[:, None], a]
    _, _, table = ref._on(rf.device)
    tup = refine_inplane(u, enc, rf, scene["q"], rel, (n, a), lat, ref, k=5)
    cen = {"D": torch.eye(3, device="cuda").expand(3, KEEP, 3, 3).contiguous(), "seed": n, "cossin": table[a]}
    dic = refine_inplane(u, enc, rf, scene["q"], rel, cen, lat, ref, k=5)
    for key in tup:
        assert (torch.equal(tup[key], dic[key]) if torch.is_tensor(tup[key]) else tup[key] == dic[key]), key


def test_track_inplane_scores_and_seeds(gpu_model, grids, scene):
    from nope_b200.inplane_refine import propose
    from nope_b200.track import seed_centres, track_inplane
    u, ref, rel = gpu_model.u_net, grids["ref"], grids["rel"]
    enc = u.encoder
    u.set_metric("l2")
    rf = enc.encode_image(scene["r"])
    P = 3
    prior = torch.from_numpy(to.random_rotations(3 * P, np.random.default_rng(4)).reshape(3, P, 3, 3)).cuda()
    out = track_inplane(u, enc, rf, scene["q"], rel, prior, ref, k=5)
    assert out["D"].shape == (3, 5, 3, 3) and out["score"].shape == (3, 5)
    assert out["hypotheses"] == ref.steps * P * 9 and out["crops"] == ref.steps * P * 2
    sc = torch.stack([u.sweep(rf, out["rel6d"][:, t:t + 1], query_feat=out["latent"][:, t], want_emb=False,
                              want_sim=True)["sim"][:, 0] for t in range(5)], dim=1)
    assert torch.equal(sc, out["score"])
    # each seed swept as is: its centre pose slot against its rolled crop's latent
    cen = seed_centres(prior, ref)
    idx = torch.arange(3, device="cuda", dtype=torch.int32)[:, None].expand(3, P).reshape(-1)
    lat = enc.encode_image_rotated(scene["q"], idx, cen["cossin"].reshape(-1, 2)).view(3, P, *rf.shape[1:])
    stencils, _, _ = ref._on(rf.device)
    cand = propose(cen["D"].reshape(3, P, 9).contiguous(), cen["seed"], cen["cossin"], rel, stencils[0],
                   ref.rolls[0], 1)
    seeds = torch.stack([u.sweep(rf, cand["poses"][:, p * 9:p * 9 + 1], query_feat=lat[:, p], want_emb=False,
                                 want_sim=True)["sim"][:, 0] for p in range(P)], dim=1)
    print(f"track_inplane: best seed {seeds.max(dim=1).values.tolist()}, refined {out['score'][:, 0].tolist()}")
    assert (out["score"][:, 0] >= seeds.max(dim=1).values).all()


# ------------------------------------------------------------------ track_pose_frames and PoseTracker
@pytest.fixture(scope="module")
def frame_scene():
    """three detections of two objects (91: box, 92: sphere) in two frames, detections 0 and 1 in frame 0; a bank of
    objects 91, 92 and 93 (no detection) over the 42-pose grid"""
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from nope_b200.vsd import render_depth
    from oracle import inputs
    meshes = {91: make_mesh("box"), 92: make_mesh("sphere")}
    ids = [91, 92, 91]
    rng = np.random.default_rng(8)
    spots = [(150.0, 130.0, 700.0), (560.0, 380.0, 900.0), (400.0, 250.0, 600.0)]
    R = np.stack([rot(rng) for _ in ids])
    t = np.stack([np.linalg.solve(K3, [u, v, 1.0]) * z for u, v, z in spots])
    masks = torch.stack([(render_depth(meshes[i][0], torch.from_numpy(pose(R[b], t[b])), K3, (H, W))[0] > 0)
                         .to(torch.uint8) * 255 for b, i in enumerate(ids)])
    rgb = lambda m: m[..., None].expand(*m.shape, 3).contiguous()     # noqa: E731
    frames = torch.stack([rgb(masks[0] | masks[1]), rgb(masks[2])])
    _, ref = inputs.make_images(seed=4, batch=3)
    return {"meshes": meshes, "ids": ids, "masks": masks, "frames": frames, "fi": torch.tensor([0, 0, 1]),
            "ref": ref.cuda(), "rel": synthetic_pose_batch(42, 3)[0].cuda(),
            "tp": torch.from_numpy(icosphere_object_rotations(0)), "bank_ids": [91, 92, 93]}


@pytest.fixture(scope="module")
def tracked(gpu_model, frame_scene):
    """the model with the scene's objects, its bank and a refiner over the 42-pose grid"""
    from nope_b200.inplane_refine import InplaneRefiner
    fs = frame_scene
    with_objects(gpu_model, fs["meshes"])
    bank = gpu_model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
    return gpu_model, bank, InplaneRefiner(fs["tp"], angles=A, steps=2)


def _chain(model, fs, prior, refiner, refine, occluders, bank=None):
    """frame_crops -> to_crop -> track_inplane -> pose_rotations -> to_camera -> estimate_translation (->
    refine_pose_contour), by hand"""
    from nope_b200 import contour_refine, translation
    from nope_b200.crop import detection_occluders, frame_crops, to_camera, to_crop
    from nope_b200.inplane_refine import pose_rotations
    from nope_b200.track import track_inplane
    ids, masks, fi = fs["ids"], fs["masks"], fs["fi"]
    d = np.array([fs["meshes"][i][1] for i in ids])
    crops, t0, Rv, _ = frame_crops(fs["frames"], masks, K3, d, frame_idx=fi)
    Rpc = to_crop(prior, Rv)
    u = model.u_net
    if bank is not None:
        slots = torch.tensor(bank.slots(ids), device="cuda")
        rf, rel = bank.reference_latents[slots], bank.all_relativeR[slots]
    else:
        rf, rel = u.encoder.encode_image(fs["ref"]), fs["rel"]
    out = track_inplane(u, u.encoder, rf, crops, rel, Rpc, refiner, k=K)
    R_crop = pose_rotations(out["D"], out["seed"], out["cossin"], refiner)
    R = to_camera(R_crop, Rv)
    occ = detection_occluders(masks.cuda(), fi, num_frames=2) if occluders else None
    t = torch.empty(3, K, 3, dtype=torch.float64, device="cuda")
    iou = torch.empty(3, K, dtype=torch.float64, device="cuda")
    R_out = R.clone()
    for i in sorted(set(ids)):
        rows = [b for b, j in enumerate(ids) if j == i]
        mesh = fs["meshes"][i][0]
        o = None if occ is None else occ[rows]
        tt, ii = translation.estimate_translation(mesh, R[rows], K3, masks[rows], t_init=t0[rows], occluders=o)
        if refine:
            R_out[rows], tt, fit = contour_refine.refine_pose_contour(mesh, R[rows], tt, K3, masks[rows], occluders=o)
            ii = fit["iou"]
        t[rows], iou[rows] = tt, ii
    return {"R": R_out, "t": t, "score": out["score"], "iou": iou, "R_crop": R_crop, "t0": t0, "crops": crops}


def _first(model, fs, bank, refiner, **kw):
    return model.predict_pose_frames(fs["frames"], fs["masks"], K3, fs["ids"], k=K, refiner=refiner,
                                     frame_idx=fs["fi"], bank=bank, **kw)


@pytest.mark.parametrize("with_bank", [True, False])
@pytest.mark.parametrize("refine,occluders", [(None, None), ("contour", None), ("contour", "detections")])
def test_track_pose_frames_equals_the_chain(tracked, frame_scene, with_bank, refine, occluders):
    model, bank, refiner = tracked
    fs = frame_scene
    prior = _first(model, fs, bank, refiner)["R"][:, :KEEP]
    src = dict(bank=bank) if with_bank else dict(reference=fs["ref"], all_relativeR=fs["rel"], template_poses=fs["tp"])
    out = model.track_pose_frames(fs["frames"], fs["masks"], K3, fs["ids"], prior, refiner, k=K, refine=refine,
                                  frame_idx=fs["fi"], occluders=occluders, **src)
    ref = _chain(model, fs, prior, refiner, refine, occluders, bank if with_bank else None)
    for key in ("R", "t", "score", "iou", "R_crop", "t0", "crops"):
        assert torch.equal(out[key], ref[key]), key
    assert set(out) == set(ref)


def test_synchronisations(tracked, frame_scene):
    """track_pose_frames synchronises as often as predict_pose_frames (with the bank and with references);
    PoseTracker.step with min_iou = 0 as often as track_pose_frames, and once more with the lost check"""
    from nope_b200.track import PoseTracker
    model, bank, refiner = tracked
    fs = frame_scene
    args = (fs["frames"], fs["masks"], K3, fs["ids"])
    prior = _first(model, fs, bank, refiner)["R"][:, :KEEP]
    refs = dict(reference=fs["ref"], all_relativeR=fs["rel"], template_poses=fs["tp"])
    counts = {}
    for name, src in (("bank", dict(bank=bank)), ("references", dict(refs))):
        search = lambda: model.predict_pose_frames(*args, k=K, refiner=refiner, frame_idx=fs["fi"], **src)  # noqa
        track = lambda: model.track_pose_frames(*args, prior, refiner, k=K, frame_idx=fs["fi"], **src)     # noqa
        search(), track()                                                                # warm-up
        _, counts[f"search {name}"] = count_host_syncs(search)
        _, counts[f"track {name}"] = count_host_syncs(track)
    tr0 = PoseTracker(model, bank, refiner, keep=KEEP, k=K, min_iou=0.0)
    tr1 = PoseTracker(model, bank, refiner, keep=KEEP, k=K, min_iou=1e-9)
    for tr in (tr0, tr1):
        tr.step(*args, [1, 2, 3], frame_idx=fs["fi"])
        tr.step(*args, [1, 2, 3], frame_idx=fs["fi"])                                    # warm-up of the tracked path
    out0, counts["step min_iou=0"] = count_host_syncs(lambda: tr0.step(*args, [1, 2, 3], frame_idx=fs["fi"]))
    out1, counts["step min_iou>0"] = count_host_syncs(lambda: tr1.step(*args, [1, 2, 3], frame_idx=fs["fi"]))
    print(f"syncs: {counts}")
    assert out0["tracked"].all() and out1["tracked"].all()
    assert counts["track bank"] == counts["search bank"]
    assert counts["track references"] == counts["search references"]
    assert counts["step min_iou=0"] == counts["track bank"]
    assert counts["step min_iou>0"] == counts["track bank"] + 1


@pytest.mark.parametrize("refine,occluders", [(None, None), ("contour", "detections")])
def test_pose_tracker_rows(tracked, frame_scene, refine, occluders):
    from nope_b200.crop import detection_occluders
    from nope_b200.track import PoseTracker
    model, bank, refiner = tracked
    fs = frame_scene
    args = (fs["frames"], fs["masks"], K3)
    ids, fi = fs["ids"], fs["fi"]
    occ = detection_occluders(fs["masks"], fi, num_frames=2) if occluders else None
    tr = PoseTracker(model, bank, refiner, keep=KEEP, k=K, min_iou=0.0, refine=refine, occluders=occluders)

    def same(a, b, rows=None, skip=("tracked",)):
        for key in b:
            if key not in skip:
                x = a[key] if rows is None else a[key][rows]
                assert torch.equal(x, b[key]), key

    # frame 1: every id is new -> the refined bank search
    out1 = tr.step(*args, ids, [10, 11, 12], frame_idx=fi)
    same(out1, _first(model, fs, bank, refiner, refine=refine, occluders=occluders))
    assert not out1["tracked"].any() and set(tr.tracks) == {10, 11, 12}
    # frame 2: all tracked from frame 1's R[:, :keep]
    out2 = tr.step(*args, ids, [10, 11, 12], frame_idx=fi)
    want = model.track_pose_frames(*args, ids, out1["R"][:, :KEEP], refiner, bank=bank, k=K, refine=refine,
                                   frame_idx=fi, occluders=occluders)
    same(out2, want)
    assert out2["tracked"].all()
    # frame 3: 12 dropped, 13 new (row 2 searched on its own), 10 and 11 tracked from frame 2
    out3 = tr.step(*args, ids, [10, 11, 13], frame_idx=fi)
    assert out3["tracked"].tolist() == [True, True, False] and set(tr.tracks) == {10, 11, 13}
    o = None if occ is None else occ[[0, 1]]
    want = model.track_pose_frames(fs["frames"], fs["masks"][[0, 1]], K3, ids[:2], out2["R"][:2, :KEEP], refiner,
                                   bank=bank, k=K, refine=refine, frame_idx=fi[[0, 1]], occluders=o)
    same(out3, want, [0, 1])
    o = None if occ is None else occ[[2]]
    want = model.predict_pose_frames(fs["frames"], fs["masks"][[2]], K3, ids[2:], k=K, refiner=refiner,
                                     refine=refine, frame_idx=fi[[2]], occluders=o, bank=bank)
    same(out3, want, [2])
    # frame 4: rows below the IoU threshold are lost and searched again
    prior = out3["R"][:, :KEEP]
    trial = model.track_pose_frames(*args, ids, prior, refiner, bank=bank, k=K, refine=refine, frame_idx=fi,
                                    occluders=occluders)
    best = trial["iou"].amax(dim=1)
    tr.min_iou = float(best.median())
    lost = [b for b in range(3) if not bool(best[b] >= tr.min_iou)]
    out4 = tr.step(*args, ids, [10, 11, 13], frame_idx=fi)
    print(f"best IoU {best.tolist()}, min_iou {tr.min_iou}, lost rows {lost}")
    assert out4["tracked"].tolist() == [b not in lost for b in range(3)] and 1 <= len(lost) < 3
    keptr = [b for b in range(3) if b not in lost]
    same(out4, {key: v[keptr] for key, v in trial.items()}, keptr)
    o = None if occ is None else occ[lost]
    want = model.predict_pose_frames(fs["frames"], fs["masks"][lost], K3, [ids[b] for b in lost], k=K,
                                     refiner=refiner, refine=refine, frame_idx=fi[lost], occluders=o, bank=bank)
    same(out4, want, lost)
    # an id whose object changes is refused, and nothing is forgotten
    with pytest.raises(ValueError, match="changed obj_id"):
        tr.step(*args, [92, 92, 91], [10, 11, 13], frame_idx=fi)
    assert set(tr.tracks) == {10, 11, 13}


# ------------------------------------------------------------------ roll tracking through a stub engine
class StubEngine:
    """sweep() scores every pose against one template, the encoder latent of image I: a score that depends on the
    roll of the query latent only (minus the mean squared difference)"""

    def __init__(self, template):
        self.t = template
        self.device = template.device

    def sweep(self, ref_feat, poses, query_feat=None, want_emb=False, want_sim=True, k=0):
        qf = query_feat if query_feat.dim() == 5 else query_feat[:, None]
        s = -((qf - self.t) ** 2).mean(dim=(-3, -2, -1))
        sim = s[..., None].expand(*s.shape, poses.shape[1]).contiguous()
        return {"sim": sim if query_feat.dim() == 5 else sim[:, 0], "emb": None, "topv": None, "topi": None}


def _disc_image(g, size=256):
    """smooth asymmetric content inside the inscribed circle, -1 outside: rotations about the centre lose nothing"""
    ys, xs = torch.meshgrid(torch.arange(size, dtype=torch.float64), torch.arange(size, dtype=torch.float64),
                            indexing="ij")
    c = (size - 1) / 2
    img = torch.zeros(3, size, size, dtype=torch.float64)
    for ch in range(3):
        for _ in range(6):
            px, py = (torch.rand(2, generator=g, dtype=torch.float64) * 0.9 - 0.45) * size + c
            sig = float(torch.rand(1, generator=g, dtype=torch.float64)) * 18 + 8
            img[ch] += torch.exp(-((xs - px) ** 2 + (ys - py) ** 2) / (2 * sig * sig))
    img = img / img.amax(dim=(1, 2), keepdim=True) * 1.8 - 0.9
    inside = (xs - c) ** 2 + (ys - c) ** 2 <= (c - 2) ** 2
    return torch.where(inside, img, torch.tensor(-1.0, dtype=torch.float64)).float()


def test_roll_tracking_with_a_stub_engine(gpu_model, grids):
    """One image rotated by off-bin angles beta_t = beta_0 + t delta over 48 frames; frame 0 is the refined in-plane
    search, every later frame track_inplane from the previous frame's top-keep rotations.  The stub's templates
    ignore the pose, so only the roll can be right.  Measured on an H100 80GB HBM3 (700 W power limit): first frame
    0.173 degrees, tracked frames median 0.148 (max 0.323); the gates leave about twice that."""
    from nope_b200.inplane_refine import InplaneRefiner, pose_rotations, refine_inplane, roll_degrees, rotate_pairs
    from nope_b200.track import track_inplane
    enc = gpu_model.u_net.encoder
    g = torch.Generator().manual_seed(6)
    I = _disc_image(g).cuda()[None]
    stub = StubEngine(enc.encode_image(I))
    ref = InplaneRefiner(grids["R"], angles=36, steps=4)
    rel = grids["rel"][:1]
    rf = torch.zeros(1, enc.latent_dim, 32, 32, device="cuda")
    T, delta, beta0 = 48, 3.7, float(torch.rand(1, generator=g, dtype=torch.float64)) * 360 - 180
    beta = beta0 + delta * torch.arange(T, dtype=torch.float64)
    cs = torch.stack([torch.cos(torch.deg2rad(-beta)), torch.sin(torch.deg2rad(-beta))], dim=-1).float()
    imgs = rotate_pairs(I, torch.zeros(T, dtype=torch.int32).cuda(), cs.cuda())       # [T, 3, 256, 256]
    qf = enc.encode_image_inplane(imgs[:1], ref.angles)                                  # frame 0: the search
    sim = stub.sweep(rf, rel, qf.view(1, ref.angles, *qf.shape[2:]))["sim"].view(1, -1)
    flat = torch.sort(-sim, dim=1, stable=True).indices[:, :KEEP]
    n, a = flat % 642, flat // 642
    out = refine_inplane(stub, enc, rf, imgs[:1], rel, (n, a), qf[0, a[0]][None], ref, k=KEEP)
    alpha = [float(roll_degrees(out["cossin"][0, 0]))]
    for t in range(1, T):
        prior = pose_rotations(out["D"], out["seed"], out["cossin"], ref)                # [1, keep, 3, 3]
        out = track_inplane(stub, enc, rf, imgs[t:t + 1], rel, prior, ref, k=KEEP)
        alpha.append(float(roll_degrees(out["cossin"][0, 0])))
    err = ((torch.tensor(alpha, dtype=torch.float64) - beta + 180) % 360 - 180).abs()
    print(f"roll tracking over {T} frames, delta = {delta} deg, A = 36, keep = {KEEP}, {ref.steps} steps: first frame "
          f"{float(err[0]):.3f} deg, tracked median {float(err[1:].median()):.3f} deg (max {float(err[1:].max()):.3f})")
    assert float(err[1:].median()) < 0.3 and float(err[1:].max()) < 0.65
