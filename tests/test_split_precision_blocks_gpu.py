"""The split-precision engines one module at a time: every block of the template encoder (csrc/encoder.cuh), the SD VAE
encoder and the SD VAE decoder (csrc/vae.cuh) run on its own through the engines' run_block entry points, fed the
float64 oracle's input to that module and compared with the oracle's output of it.

The end-to-end checks (test_unet_gpu.py, test_vae_gpu.py, test_vae_decoder_gpu.py) leave 3-5x headroom over their
measured error, and a one-layer fault of fp16 size (a tap's A_lo segment lost, the residual's lo half ignored, an
out_lo row written to the wrong pixel) adds ~1e-4 at its layer, which later GroupNorms and residual sums dilute.  Per
module, split precision is ~1e-5 and fp16 operands are ~2e-4, so the gate below separates the two, and a failure
names the module.

The module list is checked against the engines' weight schemas on the CPU, so no layer escapes."""
import ctypes as C

import pytest
import torch

from _util import (DEC_CHUNK, ENC_CHUNK, ENC_MODULES, SPLIT_BLOCK_TOL, VAE_CHUNK, VAE_MODULES, encoder_taps,
                   encoder_weights, log, mixed_images, pair_tiles, pick_bn, rounds, run_block, skip_without_gpu,
                   vae_encoder_taps, worst_block_rel_l2)


DEC_MODULES = (["decoder.conv_in", "decoder.mid_block.resnets.0", "decoder.mid_block.attentions.0",
                "decoder.mid_block.resnets.1"]
               + [m for i in range(4) for m in [f"decoder.up_blocks.{i}.resnets.{j}" for j in range(3)]
                  + ([f"decoder.up_blocks.{i}.upsamplers.0"] if i < 3 else [])]
               + ["decoder.conv_out"])

# weight-key prefixes of the modules that own more than their own name's keys: the folds of the engines
OWNS = {"stem": ("backbone.conv1.", "backbone.bn1."),
        "encoder.conv_out": ("encoder.conv_norm_out.", "encoder.conv_out.", "quant_conv."),
        "decoder.conv_in": ("post_quant_conv.", "decoder.conv_in."),
        "decoder.conv_out": ("decoder.conv_norm_out.", "decoder.conv_out.")}

# one module per distinct path: stride 2 + downsample, the planar level, the K-segment shortcut, the planar
# shortcut, the folded upsample and its repack, the attention core
SENSITIVE = ["backbone.layer2.0", "encoder.down_blocks.0.resnets.0", "encoder.down_blocks.1.resnets.0",
             "decoder.up_blocks.3.resnets.0", "decoder.up_blocks.2.upsamplers.0", "encoder.mid_block.attentions.0"]


def _owners(key, modules):
    return [m for m in modules if key.startswith(OWNS.get(m, (m + ".",)))]


# ------------------------------------------------------------------ CPU: the module lists cover the weights
@pytest.mark.parametrize("engine", ["encoder", "vae", "decoder"])
def test_every_weight_belongs_to_exactly_one_module(engine):
    from nope_b200.synth_weights import encoder_param_shapes
    from nope_b200.vae import _vae_block_out, vae_decoder_param_shapes, vae_param_shapes
    from nope_b200.encoder import _encoder_block_out
    if engine == "encoder":
        # backbone.fc is part of the reference's state_dict, unused by its forward, and not loaded by the engine
        keys, modules = [k for k in encoder_param_shapes() if not k.startswith("backbone.fc.")], ENC_MODULES
        assert all(_encoder_block_out(m, 8) != (1, 1, 1) for m in modules)
    else:
        keys = list((vae_param_shapes if engine == "vae" else vae_decoder_param_shapes)())
        modules = VAE_MODULES if engine == "vae" else DEC_MODULES
        assert all(_vae_block_out(m) != (1, 1, 1) for m in modules)
    assert len(set(modules)) == len(modules)
    for k in keys:
        assert len(_owners(k, modules)) == 1, (k, _owners(k, modules))
    for m in modules:
        assert any(_owners(k, [m]) for k in keys), m


def test_oracle_taps_chain_the_modules():
    """each module's tapped input is the previous module's tapped output, and the last output is the result"""
    from oracle import unet_oracle, vae_oracle
    from nope_b200.synth_weights import make_encoder_state_dict, make_vae_state_dict
    import vae_decoder_oracle
    g = torch.Generator().manual_seed(3)
    x = torch.rand((1, 3, 64, 64), generator=g) * 2 - 1
    runs = []
    taps = {}
    out = unet_oracle.encode_image({k: v.double() for k, v in make_encoder_state_dict(0).items()}, x.double(),
                                   taps=taps)
    runs.append((taps, ENC_MODULES, x, out))
    sd = make_vae_state_dict(seed=0, decoder=True)
    taps = {}
    out = vae_oracle.encode(sd, x, taps=taps)
    runs.append((taps, VAE_MODULES, x, out))
    assert set(taps) >= {"down0", "down1", "down2", "down3", "mid"} and taps["mid"] is taps[VAE_MODULES[-2]][1]
    z = torch.rand((1, 4, 4, 4), generator=g)
    taps = {}
    out = vae_decoder_oracle.decode(sd, z, taps=taps)
    runs.append((taps, DEC_MODULES, z, out))
    assert set(taps) >= {"mid", "up0", "up1", "up2", "up3"}
    for taps, modules, inp, out in runs:
        assert torch.equal(taps[modules[0]][0], inp.double())
        for a, b in zip(modules, modules[1:]):
            assert taps[b][0] is taps[a][1], b
        assert taps[modules[-1]][1] is out


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def enc_sd(seeded_state_dict):
    return encoder_weights(seeded_state_dict)


@pytest.fixture(scope="module")
def encoder(enc_sd):
    skip_without_gpu()
    from nope_b200.encoder import FeatureExtractor
    fe = FeatureExtractor(descriptor_size=8).cuda()
    fe.load_state_dict(enc_sd)
    return fe


@pytest.fixture(scope="module")
def enc_taps(enc_sd):
    return encoder_taps(enc_sd)


@pytest.fixture(scope="module")
def vae_sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0, decoder=True)


@pytest.fixture(scope="module")
def vae(vae_sd):
    skip_without_gpu()
    from nope_b200.vae import VAE_StableDiffusion
    return VAE_StableDiffusion(device="cuda:0", name="VAE").load_state_dict(vae_sd)


@pytest.fixture(scope="module")
def vae_taps(vae_sd):
    return vae_encoder_taps(vae_sd)


@pytest.fixture(scope="module")
def dec_taps(vae_sd, vae):
    skip_without_gpu()
    import vae_decoder_oracle
    taps = {}
    vae_decoder_oracle.decode(vae_sd, vae.encode_image(mixed_images(DEC_CHUNK, 72).cuda()).double(), taps=taps)
    return taps


def _check_module(engine, taps, name, n, tag):
    x, ref = taps[name]
    out, pair = run_block(engine, name, x[:n].float())
    assert out.shape == ref[:n].shape
    e, img = worst_block_rel_l2(out, ref[:n])
    co, ho = ref.shape[1], ref.shape[2]
    log("split_block", engine=tag, module=name, n=n, rel_l2=e, worst_image=img,
        rounds=rounds(pair_tiles(n, ho, ho, (co + 63) // 64 * 64, pick_bn((co + 63) // 64 * 64)), out.device))
    assert e <= SPLIT_BLOCK_TOL, (name, n, e)
    if pair is not None:
        # the (hi, lo) copy of the stream is the fp32 stream split in two: |hi + lo - x| <= 2^-21 |x| + 2^-24
        bad = (pair.double() - out.double()).abs() > out.double().abs() * 2.0 ** -21 + 2.0 ** -24
        assert not bad.any(), (name, n, int(bad.sum()), bad.nonzero()[:4].tolist())


# ------------------------------------------------------------------ GPU: every module against the oracle
def _ns(chunk):
    return [1, 3, chunk]


@pytest.mark.gpu
@pytest.mark.parametrize("n", _ns(ENC_CHUNK))
@pytest.mark.parametrize("name", ENC_MODULES)
def test_encoder_module_matches_the_float64_oracle(encoder, enc_taps, name, n):
    _check_module(encoder, enc_taps, name, n, "encoder")


@pytest.mark.gpu
@pytest.mark.parametrize("n", _ns(VAE_CHUNK))
@pytest.mark.parametrize("name", VAE_MODULES)
def test_vae_encoder_module_matches_the_float64_oracle(vae, vae_taps, name, n):
    _check_module(vae, vae_taps, name, n, "vae")


@pytest.mark.gpu
@pytest.mark.parametrize("n", _ns(DEC_CHUNK))
@pytest.mark.parametrize("name", DEC_MODULES)
def test_vae_decoder_module_matches_the_float64_oracle(vae, dec_taps, name, n):
    _check_module(vae, dec_taps, name, n, "decoder")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 5])
def test_projector_with_padded_descriptor_sizes(enc_sd, enc_taps, D):
    """the projector's output channels are padded to 64 in the weights and the store: D = 8 and one D that is not a
    multiple of 8, on an engine that differs only in projector.3"""
    from nope_b200.encoder import FeatureExtractor
    g = torch.Generator().manual_seed(90 + D)
    sd = dict(enc_sd)
    sd["projector.3.weight"] = (torch.rand((D, 256, 1, 1), generator=g) * 2 - 1) / 16
    fe = FeatureExtractor(descriptor_size=D).cuda()
    fe.load_state_dict(sd)
    x = enc_taps["projector"][0]
    w1, w3 = enc_sd["projector.1.weight"].cuda().double(), sd["projector.3.weight"].cuda().double()
    ref = torch.nn.functional.conv2d(torch.relu(torch.nn.functional.conv2d(torch.relu(x), w1)), w3)
    for n in (1, ENC_CHUNK):
        out = fe.run_block("projector", x[:n].float())
        e, _ = worst_block_rel_l2(out, ref[:n])
        log("split_block_projector", D=D, n=n, rel_l2=e)
        assert out.shape == (n, D, 32, 32) and e <= SPLIT_BLOCK_TOL
    fe._drop_engine()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SENSITIVE)
def test_the_gate_separates_split_precision_from_fp16(encoder, vae, enc_taps, vae_taps, dec_taps, name):
    """the same input rounded to fp16 (lo = 0) misses the gate by at least 4x: a module that lost its lo operands
    would fail the module test"""
    engine, taps = (encoder, enc_taps) if name.startswith("backbone.") else (
        vae, dec_taps if name.startswith("decoder.") else vae_taps)
    x, ref = taps[name]
    n = 3
    out, _ = run_block(engine, name, x[:n].half().float())
    e, _ = worst_block_rel_l2(out, ref[:n])
    exact, _ = worst_block_rel_l2(run_block(engine, name, x[:n].float())[0], ref[:n])
    log("split_block_fp16_input", module=name, rel_l2=e, split_rel_l2=exact, margin=e / SPLIT_BLOCK_TOL)
    assert e >= 4 * SPLIT_BLOCK_TOL, (name, e)


# ------------------------------------------------------------------ GPU: argument checks
@pytest.mark.gpu
def test_argument_checks(encoder, vae):
    from nope_b200 import _lib
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    x = torch.zeros((ENC_CHUNK + 1, 256, 32, 32), device="cuda")
    out = torch.empty(1 << 26, device="cuda")

    def enc(name, C_, H, n, cap=out.numel(), h=None):
        return _lib.check(lib.nope_encoder_run_block(h or encoder._engine(x.device), name, _lib.ptr(x), C_, H, n,
                                                     _lib.ptr(out), cap, s))

    def run(fn, h, name, C_, H, n):
        return _lib.check(fn(h, name, _lib.ptr(x), C_, H, n, _lib.ptr(out), None, out.numel(), s))

    cases = [(lambda: enc(b"backbone.layer5.0", 256, 128, 1), "unknown encoder module backbone.layer5.0"),
             (lambda: enc(b"backbone.layer1.1", 64, 128, 1), r"takes \[n, 256, 128, 128\] inputs, got C = 64"),
             (lambda: enc(b"backbone.layer1.1", 256, 64, 1), "got C = 256, H = 64"),
             (lambda: enc(b"projector", 2048, 32, ENC_CHUNK + 1), r"n must be in \[1, 32\]"),
             (lambda: enc(b"projector", 2048, 32, 2, cap=8 * 1024), "output buffer too small")]
    ve, de = vae._engine(), vae._decoder()
    for fn, h, chunk, known in ((lib.nope_vae_run_block, ve, VAE_CHUNK, (b"encoder.mid_block.resnets.0", 512, 32)),
                                (lib.nope_vae_decoder_run_block, de, DEC_CHUNK,
                                 (b"decoder.mid_block.resnets.0", 512, 32))):
        cases += [(lambda fn=fn, h=h: run(fn, h, b"encoder.mid_block.resnets.2", 512, 32, 1), "unknown module"),
                  (lambda fn=fn, h=h, k=known: run(fn, h, k[0], 256, k[2], 1), "got C = 256, H = 32"),
                  (lambda fn=fn, h=h, k=known: run(fn, h, k[0], k[1], 64, 1), "got C = 512, H = 64"),
                  (lambda fn=fn, h=h, k=known, c=chunk: run(fn, h, k[0], k[1], k[2], c + 1), rf"n must be in \[1, {chunk}\]")]
    cases.append((lambda: _lib.check(lib.nope_vae_run_block(ve, b"encoder.conv_out", _lib.ptr(x), 512, 32, 1,
                                                            _lib.ptr(out), _lib.ptr(out), out.numel(), s)),
                  "has no \\(hi, lo\\) output"))
    for kind, create, fn, name in (("encoder", (8, 0), lib.nope_encoder_run_block, b"projector"),
                                   ("vae", (0,), lib.nope_vae_run_block, b"encoder.conv_out"),
                                   ("vae_decoder", (0,), lib.nope_vae_decoder_run_block, b"decoder.conv_out")):
        hh = C.c_void_p()
        _lib.check(getattr(lib, f"nope_{kind}_create")(C.byref(hh), *create))
        args = (hh, name, _lib.ptr(x), 512, 32, 1, _lib.ptr(out)) + ((out.numel(),) if kind == "encoder" else
                                                                     (None, out.numel()))
        with pytest.raises(_lib.NopeError, match="not finalized"):
            _lib.check(fn(*args, s))
        getattr(lib, f"nope_{kind}_destroy")(hh)
    for call, msg in cases:
        with pytest.raises(_lib.NopeError, match=msg):
            call()
    torch.cuda.synchronize()
