"""GPU: the Stable Diffusion VAE encoder (nope_b200.vae, csrc/vae.cuh, DESIGN.md section 16) against the float64
oracle (oracle/vae_oracle.py) on seeded weights; batch invariance across chunks; the rotated entry points bit for bit;
no host synchronisation; argument checks; and both VAE models end to end through PoseConditional."""
import math

import pytest
import torch

from _scenes import FLIPS, tless_batch
from _util import crop_like_images, log, no_host_sync, rel_l2, uniform_images

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vae_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0)


@pytest.fixture(scope="module")
def vae(vae_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.vae import VAE_StableDiffusion
    return VAE_StableDiffusion(device="cuda:0", name="VAE").load_state_dict(vae_sd)


@pytest.mark.parametrize("kind,B", [("uniform", 1), ("uniform", 3), ("crop", 1), ("crop", 3)])
def test_latents_match_the_float64_oracle(vae, vae_sd, kind, B):
    from oracle import vae_oracle
    x = (uniform_images if kind == "uniform" else crop_like_images)(B, B).cuda()
    z = vae.encode_image(x)
    ref = vae_oracle.encode(vae_sd, x.double())
    e = rel_l2(z, ref)
    log("vae_latent", kind=kind, B=B, rel_l2=e, launches=vae.last_launch_count)
    assert z.shape == (B, 4, 32, 32) and z.dtype == torch.float32
    assert e <= 1e-4


def test_batch_invariance_across_chunks(vae):
    x = torch.cat([uniform_images(5, 20), crop_like_images(6, 13)]).cuda()       # 33 images: two full chunks and one
    z = vae.encode_image(x)
    for b in range(33):
        assert torch.equal(vae.encode_image(x[b:b + 1])[0], z[b]), b


def test_encode_inplane_equals_materialised_rotations(vae):
    from nope_b200 import inplane
    x = torch.cat([crop_like_images(9, 2), uniform_images(9, 1)]).cuda()
    A = 12                                                           # 36 pairs: crosses two chunk boundaries
    z = vae.encode_image_inplane(x, A)
    rot = inplane.rotate_images(x, A).reshape(3 * A, 3, 256, 256)
    assert z.shape == (3, A, 4, 32, 32)
    assert torch.equal(z.reshape(3 * A, 4, 32, 32), vae.encode_image(rot))


def test_encode_rotated_equals_materialised_rotations(vae):
    from nope_b200.inplane_refine import rotate_pairs
    x = crop_like_images(10, 3).cuda()
    P = 19
    g = torch.Generator().manual_seed(11)
    idx = torch.randint(-1, 4, (P,), generator=g)                     # -1 and 3: out of range, all -1 crops
    ang = torch.rand(P, generator=g) * 2 * math.pi
    cs = torch.stack([torch.cos(ang), torch.sin(ang)], 1).cuda()
    z = vae.encode_image_rotated(x, idx.cuda(), cs)
    rot = rotate_pairs(x, idx.cuda(), cs)
    assert torch.equal(z, vae.encode_image(rot))


def test_no_host_sync(vae):
    x = crop_like_images(12, 2).cuda()
    idx = torch.tensor([0, 1, 1], device="cuda")
    cs = torch.tensor([[1.0, 0.0], [0.0, 1.0], [0.6, 0.8]], device="cuda")
    vae.encode_image_inplane(x, 4)          # engine and the angle table's device copy made outside the checked region
    with no_host_sync():
        vae.encode_image(x)
        vae.encode_image_inplane(x, 4)
        vae.encode_image_rotated(x, idx, cs)
    torch.cuda.synchronize()


def test_argument_checks(vae, vae_sd):
    import ctypes as C
    from nope_b200 import _lib
    from nope_b200.vae import VAE_StableDiffusion
    x = uniform_images(0, 1).cuda()
    with pytest.raises(_lib.NopeError):
        vae.encode_image(x.cpu())                                    # no CPU path
    with pytest.raises(_lib.NopeError):
        vae.encode_image(x[:, :, :128])
    with pytest.raises(NotImplementedError):
        vae.encode_image(x, mode="sample")
    with pytest.raises(ValueError):
        vae.encode_image_inplane(x, 0)
    with pytest.raises(ValueError):
        vae.encode_image_rotated(x, torch.zeros(2, dtype=torch.int32, device="cuda"), torch.zeros(3, 2, device="cuda"))
    with pytest.raises(_lib.NopeError):
        VAE_StableDiffusion(device="cuda:0").encode_image(x)           # no weights
    lib = _lib.load()
    out = torch.empty(1, 4, 32, 32, device="cuda")
    h = vae._engine()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for rc in (lib.nope_vae_encode(h, _lib.ptr(x), 0, _lib.ptr(out), s),
               lib.nope_vae_encode(h, None, 1, _lib.ptr(out), s),
               lib.nope_vae_encode(None, _lib.ptr(x), 1, _lib.ptr(out), s),
               lib.nope_vae_encode_inplane(h, _lib.ptr(x), 1, _lib.ptr(out), 361, _lib.ptr(out), s),
               lib.nope_vae_encode_rotated(h, _lib.ptr(x), 1, _lib.ptr(out), _lib.ptr(out), 0, _lib.ptr(out), s)):
        assert rc != 0
    hh = C.c_void_p()
    assert lib.nope_vae_create(C.byref(hh), 0) == 0
    t = torch.zeros(3)
    shape = (C.c_int64 * 1)(3)
    assert lib.nope_vae_load_tensor(hh, b"encoder.conv_in.bias", _lib.ptr(t), shape, 1) != 0   # wrong shape
    assert lib.nope_vae_load_tensor(hh, b"decoder.conv_in.bias", _lib.ptr(t), shape, 1) != 0   # not in the schema
    assert lib.nope_vae_finalize(hh) != 0                                                     # keys missing
    assert lib.nope_vae_encode(hh, _lib.ptr(x), 1, _lib.ptr(out), s) != 0                      # not finalized
    lib.nope_vae_destroy(hh)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ end to end through PoseConditional
@pytest.fixture(scope="module")
def ldm_model(vae_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.synth_weights import make_ldm_state_dict
    from nope_b200.vae import build_vae_model
    m = build_vae_model("ldm", device="cuda:0", chunk=256)
    sd = dict(make_ldm_state_dict(seed=0))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})      # a reference checkpoint's layout
    return m.load_state_dict(sd).eval()


@pytest.fixture(scope="module")
def base_model(vae_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.synth_weights import make_unet_state_dict
    from nope_b200.vae import build_vae_model
    m = build_vae_model("base", device="cuda:0")
    sd = dict(make_unet_state_dict(seed=0, channels=4))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})
    return m.load_state_dict(sd).eval()


def _poses(B, N=42):
    from nope_b200.poses import synthetic_pose_batch
    rel, R = synthetic_pose_batch(N, B)
    return rel, R


def test_ldm_predict_pose_from_images(ldm_model, vae_sd):
    from oracle import vae_oracle
    u = ldm_model.u_net
    q, r = crop_like_images(20, 2).cuda(), crop_like_images(21, 2).cuda()
    rel, R = _poses(2)
    rel = rel.cuda()
    # one query per reference
    Rp, idx, sim = ldm_model.predict_pose(q, r, rel, R, k=5)
    zq, zr = u.encoder.encode_image(q), u.encoder.encode_image(r)
    R2, idx2, sim2 = u.predict_pose(zq, zr, rel, R, k=5)
    assert torch.equal(idx, idx2) and torch.equal(sim, sim2) and torch.equal(Rp, R2.to(Rp.device))
    # top-1 on the oracle's latents
    oq, orr = vae_oracle.encode(vae_sd, q.double()).float(), vae_oracle.encode(vae_sd, r.double()).float()
    _, idx_o, _ = u.predict_pose(oq, orr, rel, R, k=1)
    log("vae_ldm_top1", engine=idx[:, 0].tolist(), oracle=idx_o[:, 0].tolist())
    assert idx[:, 0].tolist() == idx_o[:, 0].tolist()
    # Q queries per reference
    qq = torch.stack([q, q.flip(-1)], 1)
    _, idx3, sim3 = ldm_model.predict_pose(qq, r, rel, R, k=5)
    zqq = u.encoder.encode_image(qq.reshape(4, 3, 256, 256)).view(2, 2, 4, 32, 32)
    _, idx4, sim4 = u.predict_pose(zqq, zr, rel, R, k=5)
    assert idx3.shape == (2, 2, 5) and torch.equal(idx3, idx4) and torch.equal(sim3, sim4)
    # broadcast: Q queries against one reference
    _, idx5, sim5 = ldm_model.predict_pose(q, r[:1], rel[:1], R, k=5)
    _, idx6, sim6 = u.predict_pose(zq, zr[:1], rel[:1], R, k=5)
    assert idx5.shape == (2, 5) and torch.equal(idx5, idx6) and torch.equal(sim5, sim6)


def test_ldm_searches(ldm_model):
    from nope_b200.hierarchy import PoseHierarchy
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from nope_b200.refine import PoseRefiner
    q, r = crop_like_images(30, 1).cuda(), crop_like_images(31, 1).cuda()
    R0, R1 = icosphere_object_rotations(0), icosphere_object_rotations(1)
    rel0, rel1 = synthetic_pose_batch(42, 1)[0].cuda(), synthetic_pose_batch(162, 1)[0].cuda()
    _, idx, sim = ldm_model.predict_pose(q, r, rel0, k=3)
    _, idx_i, ang, sim_i = ldm_model.predict_pose_inplane(q, r, rel0, k=3, angles=1)
    assert torch.equal(idx_i, idx) and not ang.any() and torch.equal(sim_i[:, 0], sim)
    _, idx_i, ang, sim_i = ldm_model.predict_pose_inplane(q, r, rel0, k=3, angles=8)
    assert idx_i.shape == (1, 3) and sim_i.shape == (1, 8, 42)
    _, idx_c, sim_c = ldm_model.predict_pose_coarse_to_fine(q, r, [rel0, rel1], PoseHierarchy([R0, R1]), k=3, keep=4)
    assert idx_c.shape == (1, 3) and torch.isfinite(sim_c.gather(-1, idx_c)).all()
    R, seed, score = ldm_model.predict_pose_refined(q, r, rel0, PoseRefiner(R0, steps=2), k=2, keep=2)
    assert R.shape == (1, 2, 3, 3) and torch.isfinite(score).all()
    R, seed, alpha, score = ldm_model.predict_pose_inplane_refined(q, r, rel0, InplaneRefiner(R0, angles=8, steps=2),
                                                                   k=2, keep=2)
    assert R.shape == (1, 2, 3, 3) and torch.isfinite(score).all()


def test_base_predict_pose_from_images(base_model):
    u = base_model.u_net
    q, r = crop_like_images(40, 2).cuda(), crop_like_images(41, 2).cuda()
    rel, R = _poses(2)
    rel = rel.cuda()
    _, idx, sim = base_model.predict_pose(q, r, rel, R, k=5)
    zq, zr = u.encoder.encode_image(q), u.encoder.encode_image(r)
    out = u.sweep(zr, rel, query_feat=zq, want_emb=False, k=5)
    assert torch.equal(idx, out["topi"]) and torch.equal(sim, out["sim"])


@pytest.mark.parametrize("which", ["ldm", "base"])
def test_test_step_on_a_synthetic_shapenet_batch(which, ldm_model, base_model):
    from nope_b200.shapenet import SyntheticShapeNet
    model = ldm_model if which == "ldm" else base_model
    ds = SyntheticShapeNet("mug", n_items=2, grid=42)
    items = [ds[i] for i in range(2)]
    batch = {k: torch.stack([it[k] for it in items]) if isinstance(items[0][k], torch.Tensor) else
             [it[k] for it in items] for k in items[0]}
    out = model.test_step({"shapeNet_mug": batch}, 0)
    assert "shapeNet_mug" in out


def test_eval_bop_with_the_ldm_model(ldm_model, tmp_path):
    batch, cad, _ = tless_batch(tmp_path, symmetries=FLIPS)
    ldm_model.load_mesh(cad, obj_ids=[1])
    ldm_model.load_models_info(cad + "/models_info.json")
    out = ldm_model.eval_bop(batch, "obj01")
    assert 0.0 <= out["top 1, ar"] <= 1.0, out
