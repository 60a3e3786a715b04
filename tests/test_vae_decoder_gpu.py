"""GPU: the Stable Diffusion VAE decoder (VAE_StableDiffusion.decode_latent, csrc/vae.cuh, DESIGN.md section 17)
against the float64 oracle (tests/vae_decoder_oracle.py) on seeded weights, for latents of encoded images and of the
LDM UNet; batch invariance across chunks; no host synchronisation; PoseConditional.sample / generate_templates with
and without decoder weights; argument checks."""
import ctypes as C

import pytest
import torch

from _util import crop_like_images, log, no_host_sync, rel_l2, uniform_images

import vae_decoder_oracle as D

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def full_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0, decoder=True)


@pytest.fixture(scope="module")
def vae(full_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.vae import VAE_StableDiffusion
    return VAE_StableDiffusion(device="cuda:0", name="VAE").load_state_dict(full_sd)


def _model(which, vae_sd):
    from nope_b200.synth_weights import make_ldm_state_dict, make_unet_state_dict
    from nope_b200.vae import build_vae_model
    if which == "ldm":
        m, sd = build_vae_model("ldm", device="cuda:0", chunk=256), dict(make_ldm_state_dict(seed=0))
    else:
        m, sd = build_vae_model("base", device="cuda:0"), dict(make_unet_state_dict(seed=0, channels=4))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})       # a reference checkpoint's layout
    return m.load_state_dict(sd).eval()


@pytest.fixture(scope="module")
def ldm_model(full_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return _model("ldm", full_sd)


@pytest.fixture(scope="module")
def base_model(full_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return _model("base", full_sd)


def _latents(kind, B, vae, ldm_model):
    if kind == "uniform":
        return vae.encode_image(uniform_images(40 + B, B).cuda())
    if kind == "crop":
        return vae.encode_image(crop_like_images(50 + B, B).cuda())
    from nope_b200.poses import synthetic_pose_batch
    rel = synthetic_pose_batch(42, B)[0][:, 7].cuda()
    pred, _ = ldm_model.sample(crop_like_images(60 + B, B).cuda(), rel)
    return pred


@pytest.mark.parametrize("kind", ["uniform", "crop", "ldm"])
@pytest.mark.parametrize("B", [1, 3])
def test_images_match_the_float64_oracle(vae, full_sd, ldm_model, kind, B):
    z = _latents(kind, B, vae, ldm_model)
    assert z.shape == (B, 4, 32, 32)
    x = vae.decode_latent(z)
    ref = D.decode(full_sd, z.double())
    e = rel_l2(x, ref)
    log("vae_decoded_image", kind=kind, B=B, rel_l2=e, launches=vae.last_decode_launch_count,
        ref_std=float(ref.std()))
    assert x.shape == (B, 3, 256, 256) and x.dtype == torch.float32
    assert e <= 1e-4


def test_batch_invariance_across_chunks(vae):
    z = torch.cat([vae.encode_image(uniform_images(70, 9).cuda()), vae.encode_image(crop_like_images(71, 8).cuda())])
    x = vae.decode_latent(z)                     # 17 latents: two full chunks and one
    for b in range(17):
        assert torch.equal(vae.decode_latent(z[b:b + 1])[0], x[b]), b


def test_no_host_sync(vae, ldm_model):
    from nope_b200.poses import synthetic_pose_batch
    z = vae.encode_image(crop_like_images(80, 2).cuda())
    r = crop_like_images(81, 1).cuda()
    rel = synthetic_pose_batch(42, 1)[0].cuda()
    enc = ldm_model.u_net.encoder
    vae.decode_latent(z)                         # engines built outside the checked region
    ldm_model.sample(r, rel[:, 0])
    ldm_model.generate_templates(r, rel[:, :20])
    with no_host_sync():
        vae.decode_latent(z)
        ldm_model.sample(r, rel[:, 0])
        ldm_model.generate_templates(r, rel[:, :20])
    torch.cuda.synchronize()
    assert enc.has_decoder


@pytest.mark.parametrize("which", ["ldm", "base"])
def test_sample_and_generate_templates_decode(which, ldm_model, base_model):
    from nope_b200.poses import synthetic_pose_batch
    model = ldm_model if which == "ldm" else base_model
    enc = model.u_net.encoder
    assert enc.has_decoder
    r = crop_like_images(90, 2).cuda()
    rel = synthetic_pose_batch(42, 2)[0].cuda()
    feat, rgb = model.sample(r, rel[:, 3])
    assert feat.shape == (2, 4, 32, 32) and rgb.shape == (2, 3, 256, 256)
    assert torch.equal(rgb, torch.clamp((enc.decode_latent(feat) + 1) / 2, 0, 1))
    N = 21
    emb, images, vid = model.generate_templates(r, rel[:, :N])
    assert emb.shape == (2, N, 4, 32, 32) and images.shape == (2, N, 3, 256, 256) and vid is None
    want = torch.clamp((enc.decode_latent(emb.reshape(2 * N, 4, 32, 32)) + 1) / 2, 0, 1)
    assert torch.equal(images, want.view(2, N, 3, 256, 256))
    assert 0.0 <= float(images.min()) and float(images.max()) <= 1.0


@pytest.mark.parametrize("which", ["ldm", "base"])
def test_encoder_only_weights_return_none(which, full_sd):
    from nope_b200.poses import synthetic_pose_batch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    enc_only = {k: v for k, v in full_sd.items() if not (k.startswith("decoder.") or k.startswith("post_quant"))}
    model = _model(which, enc_only)
    assert not model.u_net.encoder.has_decoder
    r = crop_like_images(91, 1).cuda()
    rel = synthetic_pose_batch(42, 1)[0].cuda()
    feat, rgb = model.sample(r, rel[:, 0])
    assert feat.shape == (1, 4, 32, 32) and rgb is None
    emb, images, vid = model.generate_templates(r, rel[:, :20])
    assert emb.shape == (1, 20, 4, 32, 32) and images is None and vid is None
    with pytest.raises(Exception, match="missing"):
        model.u_net.encoder.decode_latent(feat)
    del model


def test_argument_checks(vae, full_sd):
    from nope_b200 import _lib
    z = torch.zeros(1, 4, 32, 32, device="cuda")
    with pytest.raises(_lib.NopeError):
        vae.decode_latent(z.cpu())                                   # no CPU path
    for bad in (torch.zeros(1, 4, 16, 16, device="cuda"), torch.zeros(1, 8, 32, 32, device="cuda"),
                torch.zeros(4, 32, 32, device="cuda"), torch.zeros(0, 4, 32, 32, device="cuda")):
        with pytest.raises(_lib.NopeError):
            vae.decode_latent(bad)
    lib = _lib.load()
    out = torch.empty(1, 3, 256, 256, device="cuda")
    h = vae._decoder()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for rc in (lib.nope_vae_decoder_decode(h, _lib.ptr(z), 0, _lib.ptr(out), s),
               lib.nope_vae_decoder_decode(h, None, 1, _lib.ptr(out), s),
               lib.nope_vae_decoder_decode(h, _lib.ptr(z), 1, None, s),
               lib.nope_vae_decoder_decode(None, _lib.ptr(z), 1, _lib.ptr(out), s)):
        assert rc != 0
    hh = C.c_void_p()
    assert lib.nope_vae_decoder_create(C.byref(hh), 0) == 0
    t = torch.zeros(3)
    shape = (C.c_int64 * 1)(3)
    assert lib.nope_vae_decoder_load_tensor(hh, b"decoder.conv_in.bias", _lib.ptr(t), shape, 1) != 0   # wrong shape
    assert lib.nope_vae_decoder_load_tensor(hh, b"encoder.conv_in.bias", _lib.ptr(t), shape, 1) != 0   # not decoder
    assert lib.nope_vae_decoder_load_tensor(hh, b"decoder.conv_out.bias", _lib.ptr(t), shape, 1) == 0
    assert lib.nope_vae_decoder_load_tensor(hh, b"decoder.conv_out.bias", None, shape, 1) != 0         # null data
    assert lib.nope_vae_decoder_finalize(hh) != 0                                                     # keys missing
    assert lib.nope_vae_decoder_decode(hh, _lib.ptr(z), 1, _lib.ptr(out), s) != 0                      # not finalized
    lib.nope_vae_decoder_destroy(hh)
    torch.cuda.synchronize()
