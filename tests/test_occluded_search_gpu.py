"""GPU: searches under occlusion (DESIGN.md section 27).  The two visibility kernels against the numpy oracle bit for
bit; every score path with all-visible maps against the entry points without a map, bit for bit; binary maps against
the float64 oracle; query-count invariance; fully hidden rows; exact recovery of a pose whose query is three quarters
another pose's template; and the searches that take hidden= against the chain of their stages.  The weights are
seeded: nothing here says how accurate a trained model is."""
import numpy as np
import pytest
import torch

import visibility_oracle as vo
from _util import crop_like_images, same_bits

pytestmark = pytest.mark.gpu

METRICS = ("l2", "cosine", "cosine_occlusion")
DEV = "cuda:0"


def _masks(seed, B=3):
    """scattered pixels, a solid rectangle and a disc: isolated taps and long edges"""
    rng = np.random.default_rng(seed)
    h = (rng.random((B, 256, 256)) < 0.003).astype(np.uint8)
    yy, xx = np.mgrid[:256, :256]
    for b in range(B):
        y0, x0 = rng.integers(0, 200, 2)
        h[b, y0:y0 + 50, x0:x0 + 37] = 1
        cy, cx, r = rng.uniform(40, 216, 3)
        h[b][(yy - cy) ** 2 + (xx - cx) ** 2 < (r / 4) ** 2] = 1
    return h


# ------------------------------------------------------------------ the two kernels
def test_crop_hidden_equals_oracle():
    from nope_b200.visibility import crop_hidden
    from oracle import crop_oracle
    rng = np.random.default_rng(3)
    cases = [c for c in crop_oracle.seeded_cases(n=48) if c["S"] == 256]
    for case in cases:
        H, W = case["frame"].shape[:2]
        occ = np.zeros((2, H, W), np.uint8)
        occ[0] = rng.random((H, W)) < 0.05
        y0, x0 = rng.integers(0, H // 2), rng.integers(0, W // 2)
        occ[1, y0:y0 + H // 3, x0:x0 + W // 3] = 255
        maps = np.stack([case["inv_map"]] * 2)
        got = crop_hidden(torch.from_numpy(occ).to(DEV), torch.from_numpy(maps)).cpu().numpy()
        assert np.array_equal(got, vo.crop_hidden(occ, maps)), case["name"]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_latent_visibility_equals_oracle(seed):
    from nope_b200.inplane import inplane_table
    from nope_b200.visibility import latent_visibility, latent_visibility_inplane
    h = _masks(seed)
    A = 36
    table = inplane_table(A)
    rng = np.random.default_rng(10 + seed)
    t = rng.uniform(0, 2 * np.pi, 20)
    arbitrary = torch.from_numpy(np.stack([np.cos(t), np.sin(t)], 1)).float()
    quarter = torch.tensor([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])
    cs = torch.cat([table, arbitrary, quarter, quarter[:2]])
    idx = torch.cat([torch.zeros(A, dtype=torch.int32), torch.from_numpy(rng.integers(0, 3, 20)).int(),
                     torch.tensor([1, 1, 1, 1, -1, 3], dtype=torch.int32)])
    hd = torch.from_numpy(h).to(DEV)
    got = latent_visibility(hd, cs, idx).cpu().numpy()
    assert np.array_equal(got, vo.latent_visibility(h, idx.numpy(), cs.numpy()))
    assert got[-2:].all()                                                     # out-of-range images: all visible
    tab = latent_visibility_inplane(hd, A).cpu().numpy()                      # the table form: tiled pairs
    assert np.array_equal(tab[0], got[:A])
    for q in range(1, 4):                                                     # quarter turns permute the map
        assert np.array_equal(got[A + 20 + q], np.rot90(got[A + 20], q))


# ------------------------------------------------------------------ the score paths
@pytest.fixture(scope="module")
def golden(golden_dir):
    g = np.load(f"{golden_dir}/level2_642_b1.npz")
    rf, qf = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["query_feat"])
    gen = torch.Generator().manual_seed(5)
    qs = torch.stack([qf[0]] + [qf[0] + 0.2 * (i + 1) * torch.randn(qf.shape[1:], generator=gen) * qf.std()
                                for i in range(3)])[None]                   # [1, 4, C, 32, 32]
    return rf, torch.from_numpy(g["all_relativeR"]), qs


@pytest.fixture(scope="module")
def fast_model(seeded_state_dict):
    from nope_b200.model import build_model
    return build_model(device=DEV, precision="parity_fast").load_state_dict(seeded_state_dict).eval()


def _random_visible(shape, seed, p=0.6):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape + (32, 32), generator=g) < p).to(torch.uint8)


@pytest.mark.parametrize("precision", ["fp16", "parity_fast"])
@pytest.mark.parametrize("metric", METRICS)
def test_all_visible_sweep_is_bit_identical(gpu_model, fast_model, golden, precision, metric):
    u = (gpu_model if precision == "fp16" else fast_model).u_net
    rf, poses, qs = golden
    try:
        u.set_metric(metric, 0.2)
        for chunk in (7, 642):
            u.set_chunk(chunk)
            for Q in (1, 4):
                q = qs[:, :Q]
                a = u.sweep(rf, poses, query_feat=q, want_emb=False, k=5)
                b = u.sweep(rf, poses, query_feat=q, want_emb=False, k=5,
                            query_visible=torch.ones((1, Q, 32, 32), dtype=torch.bool))
                for key in ("sim", "topv", "topi"):
                    assert same_bits(a[key], b[key]), (chunk, Q, key)
    finally:
        u.set_metric("l2")
        u.set_chunk(642)


@pytest.mark.parametrize("metric", METRICS)
def test_visible_sweep_scores_and_query_count(gpu_model_parity, golden, metric):
    """binary maps against the float64 oracle on the sweep's own templates, a fully hidden row, and a Q-query
    visible sweep against Q one-query sweeps"""
    u = gpu_model_parity.u_net
    rf, poses, qs = golden
    vis = _random_visible((1, 4), 1)
    vis[0, 2] = 0                                                             # row 2: nothing visible
    try:
        u.set_metric(metric, 0.2)
        out = u.sweep(rf, poses, query_feat=qs, want_emb=True, k=5, query_visible=vis)
        for q in range(4):
            one = u.sweep(rf, poses, query_feat=qs[:, q], want_emb=False, k=5, query_visible=vis[:, q])
            for key in ("sim", "topv", "topi"):
                assert same_bits(out[key][:, q], one[key]), (q, key)
    finally:
        u.set_metric("l2")
    emb = out["emb"][0].reshape(642, qs.shape[2], 1024).cpu().numpy()
    for q in (0, 1, 3):
        ref = vo.scores(qs[0, q].reshape(qs.shape[2], 1024).numpy(), emb, vis[0, q].reshape(-1).numpy(), metric)
        got = out["sim"][0, q].double().cpu().numpy()
        if metric == "cosine_occlusion":      # a per-pixel cosine at the threshold may land either side
            np.testing.assert_allclose(got, ref, atol=2e-3)
        else:
            np.testing.assert_allclose(got, ref, rtol=1e-4)
    assert torch.isnan(out["sim"][0, 2]).all()
    assert out["topi"][0, 2].tolist() == [0, 1, 2, 3, 4]                    # NaNs rank by index (nope_topk)


def test_exact_recovery(gpu_model, golden):
    """the query is pose p's template with three quarters of its latent pixels taken from a distant pose's: the plain
    sweep ranks another pose first, the visible sweep with those pixels hidden ranks p first at score -0"""
    u = gpu_model.u_net
    rf, rel, _ = golden
    emb = u.sweep(rf, rel, want_emb=True)["emb"][0]                          # [642, C, 32, 32]
    p = 100
    far = int((emb - emb[p]).flatten(1).norm(dim=1).argmax())
    q = emb[p].clone()
    q[:, 8:, :] = emb[far][:, 8:, :]                                          # rows 8..31: 3/4 of the pixels
    plain = u.sweep(rf, rel, query_feat=q[None], want_emb=False, k=1)["topi"]
    assert bool((plain[0, 0] != p).item()), "precondition: the plain sweep must not find p"
    vis = torch.zeros((1, 32, 32), dtype=torch.uint8)
    vis[:, :8, :] = 1
    out = u.sweep(rf, rel, query_feat=q[None], want_emb=False, k=1, query_visible=vis)
    assert int(out["topi"][0, 0]) == p
    v = out["topv"][0, 0]
    assert float(v) == 0.0 and torch.signbit(v)


def test_ldm_all_visible_is_bit_identical(golden_dir):
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict
    g = np.load(f"{golden_dir}/ldm_b1_n3.npz")
    ref, qry = torch.from_numpy(g["ref_latent"]), torch.from_numpy(g["query_latent"])
    poses = torch.from_numpy(g["all_relativeR"])
    m = UNetModelPose(device=DEV, chunk=2).load_state_dict(make_ldm_state_dict(seed=0))
    qs = torch.stack([qry[0], qry[0] * 0.5, qry[0] + 0.1])[None]             # Q = 3
    a = m.sweep(ref, poses, qs, want_emb=False, k=2)
    b = m.sweep(ref, poses, qs, want_emb=False, k=2, query_visible=torch.ones((1, 3, 32, 32), dtype=torch.uint8))
    for key in ("sim", "topv", "topi"):
        assert same_bits(a[key], b[key]), key
    vis = _random_visible((1, 3), 2)
    out = m.sweep(ref, poses, qs, want_emb=True, k=2, query_visible=vis)
    emb = out["emb"][0].reshape(poses.shape[1], qs.shape[2], 1024).cpu().numpy()
    for q in range(3):
        ref_s = vo.scores(qs[0, q].reshape(qs.shape[2], 1024).numpy(), emb, vis[0, q].reshape(-1).numpy(), "l2")
        np.testing.assert_allclose(out["sim"][0, q].double().cpu().numpy(), ref_s, rtol=1e-4)


@pytest.mark.parametrize("metric", METRICS)
def test_standalone_scores(metric):
    """nope_score_topk_visible with all-visible maps against nope_score_topk_grouped and score_topk against
    nope_score_topk_multi, bit for bit; binary maps against the float64 oracle"""
    from nope_b200.bank import RowPlan, score_rows
    from nope_b200.model import score_topk
    g = torch.Generator().manual_seed(4)
    O, N, A, C = 3, 50, 4, 8
    t = torch.randn(O, N, C, 32, 32, generator=g).to(DEV)
    bank = type("Bank", (), {})()
    bank.templates, bank.device, bank.num_poses = t, t.device, N
    plan = RowPlan([2, 0, 2], A, DEV)
    q = torch.randn(3, A, C, 32, 32, generator=g).to(DEV)
    ones = torch.ones((3, A, 32, 32), dtype=torch.uint8)
    a = score_rows(bank, q, plan, metric, 0.2, 5)
    b = score_rows(bank, q, plan, metric, 0.2, 5, visible=ones)
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    qf = q[:, 0]
    a = score_topk(qf, t[:1], k=5, metric=metric)
    b = score_topk(qf, t[:1], k=5, metric=metric, visible=torch.ones((3, 32, 32), dtype=torch.bool))
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    vis = _random_visible((3,), 3)
    sim, _ = score_topk(qf, t[:1], k=5, metric=metric, visible=vis)
    for r in range(3):
        ref = vo.scores(qf[r].reshape(C, 1024).cpu().numpy(), t[0].reshape(N, C, 1024).cpu().numpy(),
                        vis[r].reshape(-1).numpy(), metric)
        if metric == "cosine_occlusion":
            np.testing.assert_allclose(sim[r].double().cpu().numpy(), ref, atol=2e-3)
        else:
            np.testing.assert_allclose(sim[r].double().cpu().numpy(), ref, rtol=1e-4)


# ------------------------------------------------------------------ the searches
def _hidden_crops(B, seed):
    h = torch.from_numpy(_masks(seed, B)).bool()
    return h


def test_predict_pose_chain(gpu_model, golden):
    from nope_b200.visibility import latent_visibility
    m = gpu_model
    _, rel, _ = golden
    q, ref = crop_like_images(1, 2), crop_like_images(2, 1)
    q = q[None]                                                               # [1, Q = 2, 3, 256, 256]
    hidden = _hidden_crops(2, 4)[None]
    R0, i0, s0 = m.predict_pose(q, ref, rel, k=5)
    Rz, iz, sz = m.predict_pose(q, ref, rel, k=5, hidden=torch.zeros_like(hidden))
    assert same_bits(i0, iz) and same_bits(s0, sz)
    _, idx, sim = m.predict_pose(q, ref, rel, k=5, hidden=hidden)
    qf, rf = m._encode(q, ref, "l2")
    vis = latent_visibility(hidden[0].to(DEV), torch.tensor([[1.0, 0.0]] * 2)).view(1, 2, 32, 32)
    out = m.u_net.sweep(rf, rel, query_feat=qf, want_emb=False, k=5, query_visible=vis)
    assert same_bits(out["sim"], sim) and same_bits(out["topi"], idx)


def test_inplane_and_bank_chains(gpu_model, golden):
    from nope_b200.model import topk
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.visibility import latent_visibility_inplane
    m = gpu_model
    _, rel, _ = golden
    A = 6
    q, ref = crop_like_images(3, 2), crop_like_images(4, 1)
    hidden = _hidden_crops(2, 5)
    # predict_pose_inplane: one reference, the broadcast query form [Q, 3, 256, 256]
    base = m.predict_pose_inplane(q, ref, rel, k=5, angles=A)
    zero = m.predict_pose_inplane(q, ref, rel, k=5, angles=A, hidden=torch.zeros_like(hidden))
    for x, y in zip(base[1:], zero[1:]):
        assert same_bits(x, y)
    _, nearest, angle, sim = m.predict_pose_inplane(q, ref, rel, k=5, angles=A, hidden=hidden)
    enc = m.u_net.encoder
    rf = enc.encode_image(ref.to(DEV))
    lat = enc.encode_image_inplane(q.to(DEV), A)
    vis = latent_visibility_inplane(hidden.to(DEV), A)
    s = m.u_net.sweep(rf, rel, query_feat=lat.view(1, -1, *lat.shape[2:]), want_emb=False, want_sim=True, k=0,
                      query_visible=vis.view(1, -1, 32, 32))["sim"]
    _, top = topk(s.view(-1, A * rel.shape[1]), 5)
    assert same_bits(s.view(2, A, -1), sim) and same_bits(top % rel.shape[1], nearest)
    # the bank against retrieval_inplane with the same hidden
    tp = torch.from_numpy(icosphere_object_rotations(2))                     # the 642 poses of the level-2 grid
    bank = m.build_template_bank([7], ref, rel, tp)
    r_sim, r_near, r_ang = m.retrieval_inplane(q, bank.templates, k=5, angles=A, hidden=hidden)
    _, b_near, b_ang, b_sim = m.predict_pose_bank(q, [7, 7], bank, k=5, angles=A, hidden=hidden)
    assert same_bits(r_sim, b_sim) and same_bits(r_near, b_near) and same_bits(r_ang, b_ang)
    z_sim, _, _ = m.retrieval_inplane(q, bank.templates, k=5, angles=A, hidden=torch.zeros_like(hidden))
    p_sim, _, _ = m.retrieval_inplane(q, bank.templates, k=5, angles=A)
    assert same_bits(z_sim, p_sim)
    _, _, _, zb = m.predict_pose_bank(q, [7, 7], bank, k=5, angles=A, hidden=torch.zeros_like(hidden))
    _, _, _, pb = m.predict_pose_bank(q, [7, 7], bank, k=5, angles=A)
    assert same_bits(zb, pb)


def test_refined_scores_equal_visible_sweeps(gpu_model, golden):
    """predict_pose_inplane_refined with hidden= is refine_inplane with the same hidden, and every score it returns is
    the score a separate visible sweep gives its rel6d against its latent, with that roll's map"""
    from nope_b200.inplane_refine import InplaneRefiner, refine_inplane
    from nope_b200.poses import icosphere_object_rotations
    from nope_b200.visibility import latent_visibility, latent_visibility_inplane
    m = gpu_model
    _, rel, _ = golden
    tp = torch.from_numpy(icosphere_object_rotations(2))
    refiner = InplaneRefiner(tp, angles=6, steps=2)
    q, ref = crop_like_images(5, 2), crop_like_images(6, 1)
    hidden = _hidden_crops(2, 6)
    plain = m.predict_pose_inplane_refined(q, ref, rel, refiner, k=3)
    zero = m.predict_pose_inplane_refined(q, ref, rel, refiner, k=3, hidden=torch.zeros_like(hidden))
    for x, y in zip(plain, zero):
        assert same_bits(x, y)
    R, seed, alpha, score = m.predict_pose_inplane_refined(q, ref, rel, refiner, k=3, hidden=hidden)
    enc, u = m.u_net.encoder, m.u_net
    rf = enc.encode_image(ref.to(DEV))
    lat = enc.encode_image_inplane(q.to(DEV), 6)
    vis = latent_visibility_inplane(hidden.to(DEV), 6)
    sim = u.sweep(rf, rel, query_feat=lat.view(1, -1, *lat.shape[2:]), want_emb=False, want_sim=True, k=0,
                  query_visible=vis.view(1, -1, 32, 32))["sim"]
    from nope_b200.model import topk
    _, top = topk(sim.view(2, -1), 2)
    N = rel.shape[1]
    seed_lat = lat[torch.arange(2, device=DEV)[:, None], top // N]
    out = refine_inplane(u, enc, rf, q.to(DEV)[None], rel, ((top % N)[None], (top // N)[None]), seed_lat[None],
                         refiner, k=3, hidden=hidden[None])
    assert same_bits(out["score"][0], score) and same_bits(out["seed"][0], seed)
    _assert_visible_sweeps(u, rf.expand(2, *rf.shape[1:]), hidden.to(DEV), out)


def _assert_visible_sweeps(u, ref_rows, hidden_rows, out):
    """every score of refine_inplane's dict `out` (rows [R] once flattened) is what a separate visible sweep gives its
    rel6d against its latent, with the map latent_visibility makes of its row's hidden mask at its roll"""
    from nope_b200.visibility import latent_visibility
    k = out["score"].shape[-1]
    seed, score = out["seed"].reshape(-1, k), out["score"].reshape(-1, k)
    cs, rel6 = out["cossin"].reshape(-1, k, 2), out["rel6d"].reshape(-1, k, 6)
    lat = out["latent"].reshape(-1, k, *out["latent"].shape[-3:])
    checked = 0
    for r in range(seed.shape[0]):
        for j in range(k):
            if int(seed[r, j]) < 0:
                continue
            v = latent_visibility(hidden_rows[r:r + 1], cs[r, j][None])
            s = u.sweep(ref_rows[r:r + 1], rel6[r, j].view(1, 1, 6), query_feat=lat[r, j][None], want_emb=False,
                        want_sim=True, query_visible=v)["sim"]
            assert same_bits(s.view(()), score[r, j]), (r, j)
            checked += 1
    assert checked > 0


# ------------------------------------------------------------------ frames and tracks
@pytest.fixture(scope="module")
def occluded_frame():
    """three detections of two objects (91: box, 92: sphere) in two frames; detection 1 lies across detection 0's
    crop in frame 0, so "detections" occluders reach the first crop"""
    from _scenes import K3, H, W, make_mesh, pose, rot
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from nope_b200.vsd import render_depth
    from oracle import inputs
    meshes = {91: make_mesh("box"), 92: make_mesh("sphere")}
    ids = [91, 92, 91]
    rng = np.random.default_rng(7)
    spots = [(300.0, 250.0, 700.0), (345.0, 275.0, 600.0), (400.0, 250.0, 600.0)]
    R = np.stack([rot(rng) for _ in ids])
    t = np.stack([np.linalg.solve(K3, [u, v, 1.0]) * z for u, v, z in spots])
    masks = torch.stack([(render_depth(meshes[i][0], torch.from_numpy(pose(R[b], t[b])), K3, (H, W))[0] > 0)
                         .to(torch.uint8) * 255 for b, i in enumerate(ids)])
    rgb = lambda m: m[..., None].expand(*m.shape, 3).contiguous()     # noqa: E731
    frames = torch.stack([rgb(masks[0] | masks[1]), rgb(masks[2])])
    _, ref = inputs.make_images(seed=4, batch=3)
    return {"meshes": meshes, "ids": ids, "masks": masks, "frames": frames, "fi": torch.tensor([0, 0, 1]),
            "ref": ref.cuda(), "rel": synthetic_pose_batch(42, 3)[0].cuda(), "K": K3,
            "tp": torch.from_numpy(icosphere_object_rotations(0)), "bank_ids": [91, 92, 93]}


@pytest.mark.parametrize("with_bank", [True, False])
def test_frames_occluded_search_equals_its_chain(gpu_model, occluded_frame, with_bank):
    from _scenes import with_objects
    from _util import count_host_syncs
    from nope_b200.crop import detection_occluders, frame_crops
    from nope_b200.visibility import crop_hidden
    fs = occluded_frame
    model = with_objects(gpu_model, fs["meshes"])
    ids, masks, fi = fs["ids"], fs["masks"], fs["fi"]
    A = 6
    if with_bank:
        bank = model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
        src = {"bank": bank}
    else:
        src = {"reference": fs["ref"][:1], "all_relativeR": fs["rel"][:1], "template_poses": fs["tp"].cuda()}
    args = (fs["frames"], masks, fs["K"], ids)
    kw = dict(angles=A, k=3, frame_idx=fi, occluders="detections", **src)
    model.predict_pose_frames(*args, **kw)                                      # warm-up of both
    model.predict_pose_frames(*args, occluded_search=True, **kw)
    _, n_off = count_host_syncs(lambda: model.predict_pose_frames(*args, **kw))
    out, n_on = count_host_syncs(lambda: model.predict_pose_frames(*args, occluded_search=True, **kw))
    assert n_on == n_off, (n_on, n_off)
    d = np.array([fs["meshes"][i][1] for i in ids])
    crops, _, _, inv = frame_crops(fs["frames"], masks, fs["K"], d, frame_idx=fi)
    hidden = crop_hidden(detection_occluders(masks.cuda(), fi, num_frames=2), inv)
    assert bool(hidden[0].any())                                                # the scene's occluder reaches crop 0
    if with_bank:
        R_crop, n, a, sim = model.predict_pose_bank(crops, ids, bank, k=3, angles=A, hidden=hidden)
    else:
        R_crop, n, a, sim = model.predict_pose_inplane(crops, fs["ref"][:1], fs["rel"][:1], fs["tp"].cuda(), k=3,
                                                       angles=A, hidden=hidden)
    assert same_bits(out["R_crop"], R_crop)
    assert same_bits(out["score"], sim.reshape(3, -1).gather(1, a * sim.shape[-1] + n))


def test_tracker_occluded_search(gpu_model, occluded_frame):
    from _scenes import with_objects
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.track import PoseTracker
    fs = occluded_frame
    model = with_objects(gpu_model, fs["meshes"])
    bank = model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
    refiner = InplaneRefiner(fs["tp"], angles=6, steps=2)
    args = (fs["frames"], fs["masks"], fs["K"], fs["ids"])
    tracker = PoseTracker(model, bank, refiner, keep=2, k=3, min_iou=0.0, occluders="detections",
                          occluded_search=True)
    first = tracker.step(*args, [1, 2, 3], frame_idx=fs["fi"])
    ref = model.predict_pose_frames(*args, k=3, refiner=refiner, frame_idx=fs["fi"], occluders="detections",
                                    bank=bank, occluded_search=True)
    for key in ("R", "t", "score", "iou"):
        assert same_bits(first[key], ref[key]), key
    second = tracker.step(*args, [1, 2, 3], frame_idx=fs["fi"])
    assert second["tracked"].all()
    ref = model.track_pose_frames(*args, first["R"][:, :2], refiner, bank=bank, k=3, frame_idx=fs["fi"],
                                  occluders="detections", occluded_search=True)
    for key in ("R", "t", "score", "iou"):
        assert same_bits(second[key], ref[key]), key
    with pytest.raises(ValueError, match="needs occluders"):
        PoseTracker(model, bank, refiner, occluded_search=True)


def _frame_hidden(fs):
    """frame_crops of the scene and the crop-space masks of its "detections" occluders"""
    from nope_b200.crop import detection_occluders, frame_crops
    from nope_b200.visibility import crop_hidden
    d = np.array([fs["meshes"][i][1] for i in fs["ids"]])
    crops, t0, Rv, inv = frame_crops(fs["frames"], fs["masks"], fs["K"], d, frame_idx=fs["fi"])
    hidden = crop_hidden(detection_occluders(fs["masks"].cuda(), fs["fi"], num_frames=2), inv)
    assert bool(hidden[0].any())
    return crops, Rv, hidden


def test_bank_refined_and_tracked_scores_are_visible_sweeps(gpu_model, occluded_frame):
    """predict_pose_bank_refined(hidden=) equals refine_inplane in the detections' order (detections 0 and 2 share a
    bank slot, so the bank's group order differs), track_pose_frames(occluded_search=True) equals track_inplane with
    crop_hidden of the same occluders, and every score either returns is a separate visible sweep of its pose"""
    from _scenes import with_objects
    from nope_b200.crop import to_crop
    from nope_b200.inplane_refine import InplaneRefiner, refine_inplane
    from nope_b200.track import track_inplane
    fs = occluded_frame
    model = with_objects(gpu_model, fs["meshes"])
    u, enc = model.u_net, model.u_net.encoder
    bank = model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
    refiner = InplaneRefiner(fs["tp"], angles=6, steps=2)
    crops, Rv, hidden = _frame_hidden(fs)
    ids = fs["ids"]
    sd = torch.tensor([fs["bank_ids"].index(i) for i in ids], device=DEV)
    ref_rows, rel_rows = bank.reference_latents[sd], bank.all_relativeR[sd]
    # the bank-refined search
    _, seed, _, score = model.predict_pose_bank_refined(crops, ids, bank, refiner, k=3, keep=2, hidden=hidden)
    _, n, a, _ = model.predict_pose_bank(crops, ids, bank, k=2, angles=6, hidden=hidden)
    lat = enc.encode_image_inplane(crops, 6)
    seed_lat = lat[torch.arange(len(ids), device=DEV)[:, None], a]
    out = refine_inplane(u, enc, ref_rows, crops, rel_rows, (n, a), seed_lat, refiner, k=3, hidden=hidden)
    assert same_bits(out["score"], score) and same_bits(out["seed"], seed)
    _assert_visible_sweeps(u, ref_rows, hidden, out)
    # the tracked path, from the bank-refined poses in the real camera
    first = model.predict_pose_frames(fs["frames"], fs["masks"], fs["K"], ids, k=3, refiner=refiner,
                                      frame_idx=fs["fi"], occluders="detections", bank=bank, occluded_search=True)
    prior = first["R"][:, :2]
    tracked = model.track_pose_frames(fs["frames"], fs["masks"], fs["K"], ids, prior, refiner, bank=bank, k=3,
                                      frame_idx=fs["fi"], occluders="detections", occluded_search=True)
    out = track_inplane(u, enc, ref_rows, crops, rel_rows, to_crop(prior, Rv.to(DEV)), refiner, k=3, hidden=hidden)
    assert same_bits(out["score"], tracked["score"])
    _assert_visible_sweeps(u, ref_rows, hidden, out)
    plain = model.track_pose_frames(fs["frames"], fs["masks"], fs["K"], ids, prior, refiner, bank=bank, k=3,
                                    frame_idx=fs["fi"], occluders="detections")
    assert not same_bits(plain["score"], tracked["score"])               # the occluders reach the tracked scores


def test_retrieval_chain(gpu_model, golden):
    """retrieval(hidden=): an all-zero mask is retrieval without one, bit for bit; a mask is encode_image ->
    latent_visibility at roll (1, 0) -> score_topk(visible=)"""
    from nope_b200.model import score_topk
    from nope_b200.visibility import latent_visibility
    m = gpu_model
    rf, rel, _ = golden
    q = crop_like_images(9, 3)
    hidden = _hidden_crops(3, 9)
    templates = m.u_net.sweep(rf, rel, want_emb=True)["emb"]                   # [1, 642, C, 32, 32]
    s0, i0 = m.retrieval(q, templates, k=5)
    sz, iz = m.retrieval(q, templates, k=5, hidden=torch.zeros_like(hidden))
    assert same_bits(s0, sz) and same_bits(i0, iz)
    sim, idx = m.retrieval(q, templates, k=5, hidden=hidden)
    qf = m.u_net.encoder.encode_image(q.to(DEV), mode="mode")
    vis = latent_visibility(hidden.to(DEV), torch.tensor([[1.0, 0.0]] * 3))
    s1, i1 = score_topk(qf, templates, k=5, metric="l2", threshold=m._occlusion_threshold(), visible=vis)
    assert same_bits(sim, s1) and same_bits(idx, i1)
    assert not same_bits(sim, s0)
