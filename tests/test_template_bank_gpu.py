"""GPU: template banks (DESIGN.md section 25) on the template UNet (C = 8) and the SD VAE engines (C = 4, LDM and base
UNet).  The bank's templates against generate_templates and against a bank built one object at a time; grouped scores
against nope_score_topk_multi per detection, for every metric, with bank objects of 0, 1 and several detections in
interleaved order; predict_pose_bank against retrieval_inplane and against the sweep path; the refined search against
refine_inplane; predict_pose_frames(bank=) against its own chain; and its host synchronisations.  The weights are
seeded: nothing here says how accurate a trained model is."""
import numpy as np
import pytest
import torch

from _scenes import H, K3, W, make_mesh, pose, rot, with_objects
from _util import count_host_syncs

pytestmark = pytest.mark.gpu

IDS = (11, 22, 33, 44)
DETS = [33, 44, 33, 11, 33]           # 22: no detection, 11 and 44: one, 33: three, interleaved
A, K = 6, 4
METRICS = ("l2", "cosine", "cosine_occlusion")


def max_rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs() / b.abs().clamp_min(1e-30)).max())


@pytest.fixture(scope="module")
def vae_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0)


@pytest.fixture(scope="module")
def ldm_model(vae_sd):
    from nope_b200.synth_weights import make_ldm_state_dict
    from nope_b200.vae import build_vae_model
    m = build_vae_model("ldm", device="cuda:0", chunk=256)
    sd = dict(make_ldm_state_dict(seed=0))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})
    return m.load_state_dict(sd).eval()


@pytest.fixture(scope="module")
def base_model(vae_sd):
    from nope_b200.synth_weights import make_unet_state_dict
    from nope_b200.vae import build_vae_model
    m = build_vae_model("base", device="cuda:0")
    sd = dict(make_unet_state_dict(seed=0, channels=4))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})
    return m.load_state_dict(sd).eval()


@pytest.fixture(scope="module")
def scene():
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from oracle import inputs
    O = len(IDS)
    _, ref = inputs.make_images(seed=5, batch=O)
    g = torch.Generator().manual_seed(17)
    crops = torch.rand(len(DETS), 3, 256, 256, generator=g) * 2 - 1
    return {"ref": ref.cuda(), "rel": synthetic_pose_batch(42, O)[0].cuda(),
            "tp": torch.from_numpy(icosphere_object_rotations(0)), "crops": crops.cuda(),
            "slots": [IDS.index(i) for i in DETS]}


_banks = {}


def _model_and_bank(request, which, scene):
    model = request.getfixturevalue({"unet": "gpu_model", "ldm": "ldm_model", "base": "base_model"}[which])
    if which not in _banks:
        _banks[which] = model.build_template_bank(IDS, scene["ref"], scene["rel"], scene["tp"])
    return model, _banks[which]


class _metric:
    def __init__(self, model, metric):
        self.model, self.metric = model, metric

    def __enter__(self):
        self.old = getattr(self.model.testing_config, "similarity_metric", "l2")
        self.model.testing_config.similarity_metric = self.metric

    def __exit__(self, *exc):
        self.model.testing_config.similarity_metric = self.old


# ------------------------------------------------------------------ templates
@pytest.mark.parametrize("which", ["unet", "ldm", "base"])
def test_templates_equal_generate_templates(request, scene, which):
    model, bank = _model_and_bank(request, which, scene)
    C = model.u_net.encoder.latent_dim
    assert bank.templates.shape == (len(IDS), 42, C, 32, 32) and bank.templates.dtype == torch.float32
    assert bank.template_poses.dtype == torch.float64 and bank.obj_ids == IDS
    assert bank.nbytes >= len(IDS) * 42 * C * 4096
    for o in range(len(IDS)):
        emb = model.generate_templates(scene["ref"][o:o + 1], scene["rel"][o:o + 1])[0]
        assert torch.equal(bank.templates[o:o + 1], emb), o
        one = model.build_template_bank([IDS[o]], scene["ref"][o:o + 1], scene["rel"][o:o + 1], scene["tp"])
        assert torch.equal(one.templates, bank.templates[o:o + 1]), o
        assert torch.equal(one.reference_latents, bank.reference_latents[o:o + 1]), o


# ------------------------------------------------------------------ scores
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("which", ["unet", "ldm"])
def test_grouped_scores_equal_score_multi(request, scene, which, metric, tmp_path):
    """latent level: every detection's rows against nope_score_topk_multi on its object's templates, bit for bit;
    the joint top-k against nope_topk over the same sim; a saved and reloaded bank gives the same bits"""
    from nope_b200.bank import TemplateBank, search_bank
    from nope_b200.model import _score_multi, topk
    model, bank = _model_and_bank(request, which, scene)
    C = bank.latent_dim
    thr = model._occlusion_threshold()
    g = torch.Generator().manual_seed(3)
    q = (torch.randn(len(DETS), A, C, 32, 32, generator=g) * 0.5).cuda()
    sim, top = search_bank(bank, q, DETS, model.u_net, k=K, metric=metric, threshold=thr)
    assert sim.shape == (len(DETS), A, 42) and top.shape == (len(DETS), K)
    for d, s in enumerate(scene["slots"]):
        ref, _, _ = _score_multi(q[d].contiguous(), bank.templates[s:s + 1].contiguous(), 1, A, metric, thr)
        assert torch.equal(sim[d], ref), d
    _, ref_top = topk(sim.view(len(DETS), A * 42), K)
    assert torch.equal(top, ref_top)
    bank.save(tmp_path / "bank.pt")
    again = TemplateBank.load(tmp_path / "bank.pt", "cuda:0")
    sim2, top2 = search_bank(again, q, DETS, model.u_net, k=K, metric=metric, threshold=thr)
    assert torch.equal(sim2, sim) and torch.equal(top2, top)
    # already grouped detections take the path without a permutation
    order = sorted(range(len(DETS)), key=lambda d: scene["slots"][d])
    sim3, top3 = search_bank(bank, q[order], [DETS[d] for d in order], model.u_net, k=K, metric=metric, threshold=thr)
    assert torch.equal(sim3, sim[order]) and torch.equal(top3, top[order])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("which", ["unet", "ldm", "base"])
def test_predict_pose_bank_equals_retrieval_inplane(request, scene, which, metric):
    from nope_b200.inplane import compose
    model, bank = _model_and_bank(request, which, scene)
    enc = model.u_net.encoder
    crops = scene["crops"]
    with _metric(model, metric):
        R, n, a, sim = model.predict_pose_bank(crops, DETS, bank, k=K, angles=A)
        assert R.shape == (len(DETS), K, 3, 3) and R.dtype == torch.float64 and sim.shape == (len(DETS), A, 42)
        assert torch.equal(R, compose(bank.template_poses, n, a, A))
        batch = enc.encode_image_inplane(crops, A)
        same = 0
        for d, s in enumerate(scene["slots"]):
            if not torch.equal(enc.encode_image_inplane(crops[d:d + 1], A)[0], batch[d]):
                continue
            same += 1
            sim_r, n_r, a_r = model.retrieval_inplane(crops[d:d + 1], bank.templates[s:s + 1], k=K, angles=A)
            assert torch.equal(sim[d], sim_r[0]) and torch.equal(n[d], n_r[0]) and torch.equal(a[d], a_r[0]), d
    print(f"{which} {metric}: {same} of {len(DETS)} crops encode alike alone and in the batch")
    assert same >= 1


@pytest.mark.parametrize("which,metric", [("unet", "l2"), ("unet", "cosine_occlusion"), ("ldm", "l2")])
def test_predict_pose_bank_against_the_sweep(request, scene, which, metric):
    """against predict_pose_inplane of reference[slot], which scores inside the sweep: scores within 1e-5 relative,
    top-k equal except for swaps between entries whose scores lie within that tolerance; angles = 1 against the grid
    search"""
    model, bank = _model_and_bank(request, which, scene)
    crops, slots = scene["crops"], scene["slots"]
    ref, rel = scene["ref"][slots], scene["rel"][slots]
    with _metric(model, metric):
        for angles in (A, 1):
            R, n, a, sim = model.predict_pose_bank(crops, DETS, bank, k=K, angles=angles)
            R_s, n_s, a_s, sim_s = model.predict_pose_inplane(crops, ref, rel, scene["tp"], k=K, angles=angles)
            assert max_rel(sim, sim_s) < 1e-5
            flat_s = sim_s.reshape(len(DETS), -1)
            got = flat_s.gather(1, a * 42 + n)
            want = flat_s.gather(1, a_s * 42 + n_s)
            assert ((got - want).abs() <= 1e-5 * want.abs()).all()
            print(f"{which} {metric} A={angles}: max rel {max_rel(sim, sim_s):.2e}, top-k equal rows "
                  f"{int(((n == n_s) & (a == a_s)).all(1).sum())} of {len(DETS)}")
            if angles == 1:
                _, n_g, sim_g = model.predict_pose(crops, ref, rel, scene["tp"], k=K)
                assert max_rel(sim[:, 0], sim_g) < 1e-5


def test_refined_search_equals_refine_inplane(request, scene):
    from nope_b200.inplane_refine import InplaneRefiner, pose_rotations, refine_inplane, roll_degrees
    model, bank = _model_and_bank(request, "unet", scene)
    enc = model.u_net.encoder
    crops, slots = scene["crops"], scene["slots"]
    refiner = InplaneRefiner(scene["tp"], angles=A, steps=2)
    R, seed, alpha, score = model.predict_pose_bank_refined(crops, DETS, bank, refiner, k=3, keep=2)
    assert R.shape == (len(DETS), 3, 3, 3) and seed.shape == alpha.shape == score.shape == (len(DETS), 3)
    _, n, a, _ = model.predict_pose_bank(crops, DETS, bank, k=2, angles=A)
    lat = enc.encode_image_inplane(crops, A)
    seed_lat = lat[torch.arange(len(DETS), device="cuda")[:, None], a]
    sd = torch.tensor(slots, device="cuda")
    out = refine_inplane(model.u_net, enc, bank.reference_latents[sd], crops, bank.all_relativeR[sd], (n, a), seed_lat,
                         refiner, k=3)
    assert torch.equal(R, pose_rotations(out["D"], out["seed"], out["cossin"], refiner))
    assert torch.equal(seed, out["seed"]) and torch.equal(score, out["score"])
    assert torch.equal(alpha, roll_degrees(out["cossin"]))


# ------------------------------------------------------------------ predict_pose_frames
@pytest.fixture(scope="module")
def frame_scene():
    """three detections of two objects (91: box, 92: sphere) in two frames, detections 0 and 1 in frame 0; a bank of
    objects 91, 92 and 93 (no detection) over the 42-pose grid"""
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from nope_b200.vsd import render_depth
    from oracle import inputs
    meshes = {91: make_mesh("box"), 92: make_mesh("sphere")}
    ids = [91, 92, 91]
    rng = np.random.default_rng(7)
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


def _chain(model, fs, bank, refine, refiner, occluders):
    """frame_crops -> predict_pose_bank (or predict_pose_bank_refined) -> to_camera -> estimate_translation
    (-> refine_pose_contour), by hand"""
    from nope_b200 import contour_refine, translation
    from nope_b200.crop import detection_occluders, frame_crops, to_camera
    ids, masks, fi = fs["ids"], fs["masks"], fs["fi"]
    d = np.array([fs["meshes"][i][1] for i in ids])
    crops, t0, Rv, _ = frame_crops(fs["frames"], masks, K3, d, frame_idx=fi)
    if refiner is None:
        R_crop, n, a, sim = model.predict_pose_bank(crops, ids, bank, k=3, angles=A)
        score = sim.reshape(3, -1).gather(1, a * 42 + n)
    else:
        R_crop, _, _, score = model.predict_pose_bank_refined(crops, ids, bank, refiner, k=3)
    R = to_camera(R_crop, Rv)
    occ = detection_occluders(masks.cuda(), fi, num_frames=2) if occluders else None
    t = torch.empty(3, 3, 3, dtype=torch.float64, device="cuda")
    iou = torch.empty(3, 3, dtype=torch.float64, device="cuda")
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
    return {"R": R_out, "t": t, "score": score, "iou": iou, "R_crop": R_crop, "t0": t0, "crops": crops}


@pytest.mark.parametrize("refine,refined_search,occluders", [(None, False, None), ("contour", False, None),
                                                             (None, True, None), ("contour", False, "detections")])
def test_predict_pose_frames_with_a_bank_equals_the_chain(gpu_model, frame_scene, refine, refined_search, occluders):
    from nope_b200.inplane_refine import InplaneRefiner
    fs = frame_scene
    model = with_objects(gpu_model, fs["meshes"])
    bank = model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
    refiner = InplaneRefiner(fs["tp"], angles=A, steps=2) if refined_search else None
    out = model.predict_pose_frames(fs["frames"], fs["masks"], K3, fs["ids"], angles=A, k=3, refiner=refiner,
                                    refine=refine, frame_idx=fs["fi"], occluders=occluders, bank=bank)
    ref = _chain(model, fs, bank, refine, refiner, occluders)
    for key in ("R", "t", "score", "iou", "R_crop", "t0", "crops"):
        assert torch.equal(out[key], ref[key]), key


def test_frames_with_a_bank_synchronise_no_more_than_with_references(gpu_model, frame_scene):
    fs = frame_scene
    model = with_objects(gpu_model, fs["meshes"])
    bank = model.build_template_bank(fs["bank_ids"], fs["ref"], fs["rel"], fs["tp"])
    slots = [fs["bank_ids"].index(i) for i in fs["ids"]]
    tp = fs["tp"].cuda()
    args = (fs["frames"], fs["masks"], K3, fs["ids"])
    triple = (fs["ref"][slots], fs["rel"][slots], tp)
    model.predict_pose_frames(*args, *triple, angles=A, k=3, frame_idx=fs["fi"])          # warm-up
    model.predict_pose_frames(*args, angles=A, k=3, frame_idx=fs["fi"], bank=bank)
    _, n_triple = count_host_syncs(lambda: model.predict_pose_frames(*args, *triple, angles=A, k=3, frame_idx=fs["fi"]))
    out, n_bank = count_host_syncs(lambda: model.predict_pose_frames(*args, angles=A, k=3, frame_idx=fs["fi"],
                                                                     bank=bank))
    (R, n, a, sim), n_search = count_host_syncs(lambda: model.predict_pose_bank(out["crops"], fs["ids"], bank, k=3,
                                                                                angles=A))
    print(f"syncs: with references {n_triple}, with the bank {n_bank}, predict_pose_bank alone {n_search}")
    assert n_bank <= n_triple and n_search == 0
