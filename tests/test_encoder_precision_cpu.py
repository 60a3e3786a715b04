"""CPU: the encoders' precision option (DESIGN.md section 22) -- its refusals in Python and through the C ABI, which
need no GPU -- and the self-checks of the fp16-mode emulation (tests/encoder_precision_sim.py) that sets the GPU
tests' error gates."""
import ctypes as C

import pytest
import torch

import encoder_precision_sim as sim


# ------------------------------------------------------------------ Python refusals
@pytest.mark.parametrize("bad", ["fp32", "FP16", "bf16", "", None, 1])
def test_unknown_precision_is_refused(bad):
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.vae import VAE_StableDiffusion, build_vae_model
    with pytest.raises(ValueError, match="encoder precision must be one of"):
        FeatureExtractor(precision=bad)
    with pytest.raises(ValueError, match="encoder precision must be one of"):
        VAE_StableDiffusion(precision=bad)
    with pytest.raises(ValueError, match="encoder precision must be one of"):
        build_vae_model(vae_precision=bad)


def test_defaults_are_split():
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.vae import VAE_StableDiffusion
    assert FeatureExtractor().precision == "split"
    assert VAE_StableDiffusion().precision == "split"


def test_fp16_has_no_torch_or_cpu_path():
    from nope_b200 import _lib
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.vae import VAE_StableDiffusion
    with pytest.raises(_lib.NopeError, match="torch backend has none"):
        FeatureExtractor(precision="fp16", backend="torch")
    fe = FeatureExtractor(precision="fp16")            # parameters on the CPU: 'auto' would pick the torch module
    x = torch.zeros((1, 3, 256, 256))
    for call in (lambda: fe.encode_image(x), lambda: fe.encode_image_inplane(x, 4),
                 lambda: fe.encode_image_rotated(x, torch.zeros(1, dtype=torch.long), torch.zeros(1, 2))):
        with pytest.raises(_lib.NopeError, match="needs the native engine on a CUDA device"):
            call()
    with pytest.raises(_lib.NopeError, match="needs a CUDA device"):
        VAE_StableDiffusion(precision="fp16", device="cpu")
    # the split torch module on the CPU is unchanged
    assert FeatureExtractor(precision="split").encode_image(torch.zeros((1, 3, 64, 64))).shape == (1, 8, 8, 8)


# ------------------------------------------------------------------ C ABI refusals (before any CUDA call)
@pytest.mark.parametrize("kind", ["encoder", "vae"])
def test_set_option_refusals_through_the_c_abi(kind):
    from nope_b200 import _lib
    lib = _lib.load()
    fn = getattr(lib, f"nope_{kind}_set_option")
    for args, msg in (((None, b"bogus", 0), b"unknown option: bogus"),
                      ((None, None, 0), b"null option name"),
                      ((None, b"precision", 2), b"precision must be 0 (split) or 1 (fp16)"),
                      ((None, b"precision", -1), b"precision must be 0 (split) or 1 (fp16)"),
                      ((None, b"precision", 1), b"null engine")):
        assert fn(*args) != 0
        assert msg in lib.nope_last_error(), (args, lib.nope_last_error())


# ------------------------------------------------------------------ emulation self-checks
def _small_images(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((n, 3, 64, 64), generator=g) * 2 - 1


@pytest.fixture(scope="module")
def enc_sd():
    from nope_b200.synth_weights import make_encoder_state_dict
    return make_encoder_state_dict(0)


@pytest.fixture(scope="module")
def vae_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0)


def test_emulation_without_rounding_is_the_oracle(enc_sd, vae_sd):
    """rnd=False in float64 restates the float64 oracles (BatchNorm folded, conv_out and quant_conv folded)"""
    from oracle import unet_oracle, vae_oracle
    x = _small_images(2, 1)
    ref = unet_oracle.encode_image({k: v.double() for k, v in enc_sd.items()}, x.double())
    got = sim.TemplateEncoder(enc_sd, rnd=False, dtype=torch.float64).encode(x.double())
    assert sim.rel_l2(got, ref) < 1e-12
    ref = vae_oracle.encode(vae_sd, x.double())
    got = sim.VaeEncoder(vae_sd, rnd=False, dtype=torch.float64).encode(x.double())
    assert sim.rel_l2(got, ref) < 1e-12


def test_emulation_rounds_what_the_engine_stores(enc_sd, vae_sd):
    x = _small_images(2, 2)
    taps = {}
    sim.TemplateEncoder(enc_sd).encode(x, taps=taps)
    for m in sim.ENC_MODULES[:-1]:                    # every stored encoder activation is fp16 ...
        out = taps[m][1]
        assert torch.equal(out, out.half().float()), m
    proj = taps["projector"][1]                       # ... the projector's output is fp32
    assert not torch.equal(proj, proj.half().float())
    taps = {}
    sim.VaeEncoder(vae_sd).encode(x, taps=taps)
    for m in sim.VAE_MODULES:                         # the VAE's stream stays fp32
        out = taps[m][1]
        assert out.dtype == torch.float32 and not torch.equal(out, out.half().float()), m


def test_emulation_error_is_fp16_sized(enc_sd, vae_sd):
    """fp16 rounding of weights and activations: well above fp32 rounding, well below 1 %"""
    from oracle import unet_oracle, vae_oracle
    x = _small_images(2, 3)
    e = sim.rel_l2(sim.TemplateEncoder(enc_sd).encode(x),
                   unet_oracle.encode_image({k: v.double() for k, v in enc_sd.items()}, x.double()))
    assert 3e-4 < e < 1e-2, e
    e = sim.rel_l2(sim.VaeEncoder(vae_sd).encode(x), vae_oracle.encode(vae_sd, x.double()))
    assert 3e-4 < e < 1e-2, e
    # unrounded in fp32: fp32-sized
    e = sim.rel_l2(sim.VaeEncoder(vae_sd, rnd=False).encode(x), vae_oracle.encode(vae_sd, x.double()))
    assert e < 1e-5, e
