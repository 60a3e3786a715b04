"""GPU: the encoders' opt-in single-fp16 mode (precision "fp16", DESIGN.md section 22) -- the template encoder and the
SD VAE encoder -- against the float64 oracles, module by module and end to end, with gates taken from the CPU
emulation's prediction (tests/encoder_precision_sim.py); its batch, chunk and rotation invariances; its effect on an
in-plane search; and split and fp16 engines side by side in one process."""
import math

import pytest
import torch

from _util import (ENC_CHUNK, ENC_MODULES, SPLIT_BLOCK_TOL, VAE_CHUNK, VAE_MODULES, crop_like_images, encoder_taps,
                   encoder_weights, log, rel_l2, run_block, skip_without_gpu, uniform_images, vae_encoder_taps,
                   worst_block_rel_l2)

pytestmark = pytest.mark.gpu

# The emulation's prediction on the seeded weights (python tests/encoder_precision_sim.py: worst of 4 images, 2
# uniform and 2 crop-like, each module fed the float64 oracle's input; DESIGN.md section 22).  Per module:
PRED_ENC = {"stem": 2.50e-4, "backbone.layer1.0": 4.46e-4, "backbone.layer1.1": 3.45e-4, "backbone.layer1.2": 3.70e-4,
            "backbone.layer2.0": 4.18e-4, "backbone.layer2.1": 3.42e-4, "backbone.layer2.2": 3.53e-4,
            "backbone.layer2.3": 3.42e-4, "backbone.layer3.0": 4.36e-4, "backbone.layer3.1": 3.40e-4,
            "backbone.layer3.2": 3.43e-4, "backbone.layer3.3": 3.49e-4, "backbone.layer3.4": 3.42e-4,
            "backbone.layer3.5": 3.57e-4, "backbone.layer4.0": 4.41e-4, "backbone.layer4.1": 3.48e-4,
            "backbone.layer4.2": 3.46e-4, "projector": 6.59e-4}
PRED_VAE = {"encoder.conv_in": 9.4e-8, "encoder.down_blocks.0.resnets.0": 3.22e-4,
            "encoder.down_blocks.0.resnets.1": 2.81e-4, "encoder.down_blocks.0.downsamplers.0": 2.79e-4,
            "encoder.down_blocks.1.resnets.0": 4.01e-4, "encoder.down_blocks.1.resnets.1": 3.25e-4,
            "encoder.down_blocks.1.downsamplers.0": 3.07e-4, "encoder.down_blocks.2.resnets.0": 3.96e-4,
            "encoder.down_blocks.2.resnets.1": 3.18e-4, "encoder.down_blocks.2.downsamplers.0": 2.83e-4,
            "encoder.down_blocks.3.resnets.0": 3.40e-4, "encoder.down_blocks.3.resnets.1": 2.96e-4,
            "encoder.mid_block.resnets.0": 2.76e-4, "encoder.mid_block.attentions.0": 2.26e-4,
            "encoder.mid_block.resnets.1": 2.60e-4, "encoder.conv_out": 1.87e-4}
# ... and end to end, the worst image's latent rel-L2
PRED_LATENT = {"encoder": 1.54e-3, "vae": 1.09e-3}
# Gates: 2x the prediction above, and at least half of it (fp16 mode really rounds); modules whose prediction is
# below the split-precision gate (conv_in: fp32 arithmetic in both modes) are held to that gate instead.
GATE, FLOOR = 2.0, 0.5


def _module_gate(pred):
    return max(GATE * pred, SPLIT_BLOCK_TOL)


@pytest.fixture(scope="module")
def enc_sd(seeded_state_dict):
    return encoder_weights(seeded_state_dict)


@pytest.fixture(scope="module")
def enc_taps(enc_sd):
    return encoder_taps(enc_sd)


@pytest.fixture(scope="module")
def vae_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0, decoder=True)


@pytest.fixture(scope="module")
def vae_taps(vae_sd):
    return vae_encoder_taps(vae_sd)


@pytest.fixture(scope="module")
def encoder16(enc_sd):
    skip_without_gpu()
    from nope_b200.encoder import FeatureExtractor
    fe = FeatureExtractor(descriptor_size=8, precision="fp16").cuda()
    fe.load_state_dict(enc_sd)
    return fe


@pytest.fixture(scope="module")
def encoder_split(enc_sd):
    skip_without_gpu()
    from nope_b200.encoder import FeatureExtractor
    fe = FeatureExtractor(descriptor_size=8).cuda()
    fe.load_state_dict(enc_sd)
    return fe


@pytest.fixture(scope="module")
def vae16(vae_sd):
    skip_without_gpu()
    from nope_b200.vae import VAE_StableDiffusion
    return VAE_StableDiffusion(device="cuda:0", name="VAE", precision="fp16").load_state_dict(vae_sd)


@pytest.fixture(scope="module")
def vae_split(vae_sd):
    skip_without_gpu()
    from nope_b200.vae import VAE_StableDiffusion
    return VAE_StableDiffusion(device="cuda:0", name="VAE").load_state_dict(vae_sd)


# ------------------------------------------------------------------ 1. every module against the float64 oracle
def _check_module16(engine, taps, name, n, pred, tag):
    x, ref = taps[name]
    out, pair = run_block(engine, name, x[:n].float())
    assert out.shape == ref[:n].shape
    e, img = worst_block_rel_l2(out, ref[:n])
    log("fp16_block", engine=tag, module=name, n=n, rel_l2=e, worst_image=img, predicted=pred, ratio=e / pred)
    assert e <= _module_gate(pred), (name, n, e, pred)
    if pred > SPLIT_BLOCK_TOL:
        assert e >= FLOOR * pred, (name, n, e, pred)
    if tag == "encoder" and name != "projector":
        assert torch.equal(out, out.half().float()), name                  # the fp16 output, nothing below it
    if pair is not None:
        # the VAE's fp16 copy of its fp32 stream: one rounding, |hi - x| <= 2^-11 |x| (+ the subnormal step)
        bad = (pair.double() - out.double()).abs() > out.double().abs() * 2.0 ** -11 + 2.0 ** -24
        assert not bad.any(), (name, n, int(bad.sum()))
        assert torch.equal(pair, pair.half().float())


@pytest.mark.parametrize("n", [1, 3, ENC_CHUNK])
@pytest.mark.parametrize("name", ENC_MODULES)
def test_encoder_fp16_module_matches_the_float64_oracle(encoder16, enc_taps, name, n):
    _check_module16(encoder16, enc_taps, name, n, PRED_ENC[name], "encoder")


@pytest.mark.parametrize("n", [1, 3, VAE_CHUNK])
@pytest.mark.parametrize("name", VAE_MODULES)
def test_vae_fp16_module_matches_the_float64_oracle(vae16, vae_taps, name, n):
    _check_module16(vae16, vae_taps, name, n, PRED_VAE[name], "vae")


# ------------------------------------------------------------------ 2. end-to-end latents
@pytest.mark.parametrize("engine", ["encoder", "vae"])
def test_fp16_latents_match_the_prediction(engine, enc_sd, vae_sd, encoder16, encoder_split, vae16, vae_split):
    from oracle import unet_oracle, vae_oracle
    x = torch.cat([uniform_images(30, 2), crop_like_images(30, 2)]).cuda()
    if engine == "encoder":
        ref = unet_oracle.encode_image({k: v.cuda().double() for k, v in enc_sd.items()}, x.double())
        z16, zs = encoder16.encode_image(x), encoder_split.encode_image(x)
    else:
        ref = vae_oracle.encode(vae_sd, x.double())
        z16, zs = vae16.encode_image(x), vae_split.encode_image(x)
    e16, _ = worst_block_rel_l2(z16, ref)
    es, _ = worst_block_rel_l2(zs, ref)
    pred = PRED_LATENT[engine]
    log("fp16_latent", engine=engine, rel_l2_fp16=e16, rel_l2_split=es, predicted=pred, ratio_to_split=e16 / es,
        rel_l2_fp16_all=rel_l2(z16, ref))
    assert e16 <= GATE * pred and e16 >= FLOOR * pred, (e16, pred)
    assert e16 >= 10 * es, (e16, es)


# ------------------------------------------------------------------ 3. batch, chunk and rotation invariance
@pytest.mark.parametrize("engine,B", [("encoder", 33), ("vae", 17)])
def test_fp16_latent_does_not_depend_on_the_batch(engine, B, encoder16, vae16):
    enc = encoder16 if engine == "encoder" else vae16
    x = torch.cat([uniform_images(40, B - B // 2), crop_like_images(41, B // 2)]).cuda()
    z = enc.encode_image(x)
    for b in range(B):
        assert torch.equal(enc.encode_image(x[b:b + 1])[0], z[b]), b


@pytest.mark.parametrize("engine", ["encoder", "vae"])
def test_fp16_rotated_entry_points_equal_encode_of_the_rotated_batch(engine, encoder16, vae16):
    from nope_b200.inplane import rotate_images
    from nope_b200.inplane_refine import rotate_pairs
    enc = encoder16 if engine == "encoder" else vae16
    x = torch.cat([crop_like_images(42, 2), uniform_images(42, 1)]).cuda()
    A = 12                                                  # 36 pairs: crosses the chunk boundaries of both engines
    z = enc.encode_image_inplane(x, A)
    assert torch.equal(z.reshape(3 * A, *z.shape[2:]), enc.encode_image(rotate_images(x, A).reshape(3 * A, 3, 256, 256)))
    g = torch.Generator().manual_seed(43)
    P = 37
    idx = torch.randint(-1, 4, (P,), generator=g).cuda()
    ang = torch.rand(P, generator=g) * 2 * math.pi
    cs = torch.stack([torch.cos(ang), torch.sin(ang)], 1).cuda()
    assert torch.equal(enc.encode_image_rotated(x, idx, cs), enc.encode_image(rotate_pairs(x, idx, cs)))


# ------------------------------------------------------------------ 4. the in-plane search
def _standin(n_q, seed=5):
    """render-based stand-in (DESIGN.md section 14): reference and queries are shaded renders of three boxes; the
    queries at seeded off-grid viewpoints with seeded roll"""
    import numpy as np
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from inplane_refine_time import RenderEngine, three_boxes
    from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d, viewpoint_rotations
    from nope_b200.vsd import Mesh
    R2 = icosphere_object_rotations(2)
    eng = RenderEngine(None, Mesh(*three_boxes()), R2[7])
    g = np.random.default_rng(seed)
    gamma = g.uniform(-math.pi, math.pi, n_q)
    Rz = np.stack([[[math.cos(t), -math.sin(t), 0], [math.sin(t), math.cos(t), 0], [0, 0, 1]] for t in gamma])
    qR = torch.from_numpy(Rz @ viewpoint_rotations(g.standard_normal((n_q, 3)))).cuda()
    ref = eng.images(torch.from_numpy(R2[7:8]).cuda())
    return eng.images(qR), ref, relative_rotation_6d(R2, R2[7])[None].cuda()


def _score_bound(split, fp16):
    """|s_fp16 - s_split| for every (query, angle, pose) from the two modes' latents.  s = -sum_hw ||q_hw - t_hw||_4^2
    (the l2 metric), so with d = q - t and e = the change of d, per pixel | ||d + e||^2 - ||d||^2 | <= 2 ||d|| ||e|| +
    ||e||^2 (4-norms over the channels) and ||e|| <= ||dq_hw|| + ||dt_hw||: the bound is that sum over the pixels.
    split / fp16: (query latents [Q, A, C, 32, 32], templates [N, C, 32, 32]) -> [Q, A, N] float64"""
    (qs, ts), (qh, th) = split, fp16
    n4 = lambda x, dim: x.double().pow(4).sum(dim).pow(0.25)                   # noqa: E731
    eq = n4((qh - qs).flatten(3), 2)                                            # [Q, A, HW]
    et = n4((th - ts).flatten(2), 1)                                            # [N, HW]
    t = ts.flatten(2).double()
    out = []
    for i in range(qs.shape[0]):
        d = n4(qs[i].flatten(2).double()[:, None] - t[None], 2)                 # [A, N, HW]
        e = eq[i][:, None] + et[None]
        out.append((2 * d * e + e * e).sum(-1))
    return torch.stack(out)


def test_inplane_search_with_an_fp16_encoder(seeded_state_dict, enc_sd):
    """predict_pose_inplane with an fp16 encoder against the same model with a split encoder: every score moves by
    at most the bound its latents' change implies, and top-1 (angle, pose) agrees wherever the split search's margin
    between rank 1 and rank 2 exceeds twice the bound there"""
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.model import build_model
    skip_without_gpu()
    Q, A = 16, 36
    model = build_model(device="cuda:0").load_state_dict(seeded_state_dict).eval()
    split = model.u_net.encoder
    fp16 = FeatureExtractor(descriptor_size=8, precision="fp16").cuda()
    fp16.load_state_dict(enc_sd)
    q, r, rel = _standin(Q)
    out, lat = {}, {}
    for tag, enc in (("split", split), ("fp16", fp16)):
        model.u_net.encoder = enc
        out[tag] = model.predict_pose_inplane(q[None], r, rel, None, k=2, angles=A)
        rf = enc.encode_image(r)
        lat[tag] = (enc.encode_image_inplane(q, A), model.u_net.sweep(rf, rel, want_emb=True, want_sim=False)["emb"][0])
    model.u_net.encoder = split
    sim_s, sim_h = out["split"][3][0].double(), out["fp16"][3][0].double()      # [Q, A, N]
    bound = _score_bound(lat["split"], lat["fp16"])
    diff = (sim_h - sim_s).abs()
    log("fp16_inplane_scores", max_diff=float(diff.max()), max_bound=float(bound.max()),
        worst_ratio=float((diff / bound).max()), median_ratio=float((diff / bound).median()),
        latent_rel_l2=rel_l2(lat["fp16"][0], lat["split"][0]))
    assert (diff <= bound).all()
    flat = sim_s.reshape(Q, A * sim_s.shape[-1])
    top2 = flat.topk(2, dim=1)
    margin = top2.values[:, 0] - top2.values[:, 1]
    b1 = bound.reshape(Q, -1).gather(1, top2.indices[:, :1])[:, 0]
    b2 = bound.reshape(Q, -1).gather(1, top2.indices[:, 1:])[:, 0]
    clear = margin > 2 * torch.maximum(b1, b2)
    n_s, a_s = out["split"][1][0, :, 0], out["split"][2][0, :, 0]
    n_h, a_h = out["fp16"][1][0, :, 0], out["fp16"][2][0, :, 0]
    same = (n_s == n_h) & (a_s == a_h)
    log("fp16_inplane_top1", queries=Q, clear_margin=int(clear.sum()), below_margin=int((~clear).sum()),
        top1_identical=int(same.sum()), top1_identical_clear=int(same[clear].sum()))
    assert same[clear].all()


# ------------------------------------------------------------------ 5. split and fp16 engines in one process
@pytest.mark.parametrize("engine", ["encoder", "vae"])
def test_split_and_fp16_engines_side_by_side(engine, enc_sd, vae_sd, encoder16, encoder_split, vae16, vae_split):
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.vae import VAE_StableDiffusion
    x = torch.cat([uniform_images(50, 2), crop_like_images(50, 3)]).cuda()
    if engine == "encoder":
        a, h = encoder_split, encoder16
        fresh = FeatureExtractor(descriptor_size=8).cuda()
        fresh.load_state_dict(enc_sd)
    else:
        a, h = vae_split, vae16
        fresh = VAE_StableDiffusion(device="cuda:0", name="VAE").load_state_dict(vae_sd)
    za = a.encode_image(x)
    zh = h.encode_image(x)
    zh2 = h.encode_image(x)
    zf = fresh.encode_image(x)
    assert torch.equal(za, zf) and torch.equal(zh, zh2)
    assert not torch.equal(za, zh) and rel_l2(zh, za) < GATE * PRED_LATENT[engine]
    fresh._drop_engine()
