"""CPU: the SD VAE decoder's host side (nope_b200.vae): the decoder schema and the seeded recipe, the loading rules
for a complete, partial or bad decoder, checkpoint routing, the config check, the float64 oracle's folded upsample
and FLOP count (DESIGN.md section 17), and the new ABI symbols."""
import json
import os
import subprocess

import pytest
import torch

from nope_b200 import vae as V

import vae_decoder_oracle as D
from _util import SD15_CONFIG


@pytest.fixture(scope="module")
def full():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0, decoder=True)


def _decoder_keys(sd):
    return [k for k in sd if k.startswith("decoder.") or k.startswith("post_quant_conv.")]


def test_decoder_schema_counts(full):
    # 140 tensors, 49 490 199 parameters: post_quant_conv 2, conv_in 2, 2 mid resnets 16, attention 10,
    # 12 up-block resnets 96 + 2 shortcuts 4, 3 upsamplers 6, conv_norm_out 2, conv_out 2
    shapes = V.vae_decoder_param_shapes()
    assert len(shapes) == 140
    assert sum(torch.Size(s).numel() for s in shapes.values()) == 49490199
    dec = _decoder_keys(full)
    assert dec == list(shapes) and all(tuple(full[k].shape) == shapes[k] for k in dec)


def test_encoder_tensors_do_not_move_with_the_decoder(full):
    from nope_b200.synth_weights import make_vae_state_dict
    enc = make_vae_state_dict(seed=0)
    assert list(full)[:108] == list(enc) and all(torch.equal(full[k], enc[k]) for k in enc)


def test_both_attention_namings_map_to_the_same_decoder_tensors(full):
    from nope_b200.synth_weights import make_vae_state_dict
    new = make_vae_state_dict(seed=0, attention="new", decoder=True)
    assert "decoder.mid_block.attentions.0.to_out.0.weight" in new
    assert "decoder.mid_block.attentions.0.proj_attn.weight" not in new
    a, b = V.map_decoder_state_dict(full), V.map_decoder_state_dict(new)
    assert len(a) == 140 and list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    o1, o2 = D.canonical(full), D.canonical(new)
    assert set(o1) == set(o2) == set(a) and all(torch.equal(o1[k], o2[k]) for k in o1)


def test_complete_decoder_loads_and_round_trips(full):
    m = V.VAE_StableDiffusion(device="cpu").load_state_dict(full)
    assert m.has_decoder
    st = m.state_dict()
    assert len(st) == 248
    assert torch.equal(st["encoder.decoder.conv_out.weight"], full["decoder.conv_out.weight"])
    m2 = V.VAE_StableDiffusion(device="cpu").load_state_dict({k[len("encoder."):]: v for k, v in st.items()})
    assert m2.has_decoder and all(torch.equal(m2.state_dict()[k], st[k]) for k in st)


def test_partial_or_absent_decoder(full):
    enc_only = {k: v for k, v in full.items() if k not in _decoder_keys(full)}
    m = V.VAE_StableDiffusion(device="cpu").load_state_dict(enc_only)
    assert not m.has_decoder and len(m.state_dict()) == 108
    partial = dict(enc_only, **{k: full[k] for k in _decoder_keys(full)[:50]})
    m.load_state_dict(partial)
    assert not m.has_decoder and len(m.state_dict()) == 108
    with pytest.raises(Exception, match="decoder.up_blocks"):      # names the missing keys
        m._decoder()


def test_bad_decoder_entries_raise(full):
    with pytest.raises(KeyError, match="unexpected"):
        V.map_decoder_state_dict(dict(full, **{"decoder.up_blocks.4.resnets.0.conv1.bias": torch.zeros(128)}))
    with pytest.raises(KeyError, match="unexpected"):
        V.VAE_StableDiffusion(device="cpu").load_state_dict(dict(full, **{"post_quant_conv.scale": torch.zeros(1)}))
    wrong = dict(full)
    wrong["decoder.up_blocks.3.resnets.0.conv_shortcut.weight"] = torch.zeros(128, 256, 3, 3)
    with pytest.raises(ValueError, match="size mismatch"):
        V.map_decoder_state_dict(wrong)
    with pytest.raises(ValueError, match="size mismatch"):
        V.VAE_StableDiffusion(device="cpu").load_state_dict(wrong)
    both = dict(full, **{"decoder.mid_block.attentions.0.to_q.weight": full["decoder.mid_block.attentions.0.query.weight"]})
    with pytest.raises(KeyError, match="both"):
        V.map_decoder_state_dict(both)


def test_decoder_config_fields(full, tmp_path):
    V.check_decoder_config(SD15_CONFIG)
    V.check_decoder_config({k: v for k, v in SD15_CONFIG.items() if k != "out_channels"})   # default 3
    for k, v in (("out_channels", 4), ("up_block_types", ["UpDecoderBlock2D"] * 3),
                 ("up_block_types", ["AttnUpDecoderBlock2D"] * 4)):
        with pytest.raises(ValueError, match=k):
            V.check_decoder_config(dict(SD15_CONFIG, **{k: v}))
    cfg = dict(SD15_CONFIG)
    del cfg["up_block_types"]                          # diffusers' default is one block
    with pytest.raises(ValueError, match="up_block_types"):
        V.check_decoder_config(cfg)
    torch.save(full, tmp_path / "diffusion_pytorch_model.bin")
    (tmp_path / "config.json").write_text(json.dumps(SD15_CONFIG))
    assert V.VAE_StableDiffusion(pretrained_path=str(tmp_path), device="cpu").has_decoder
    (tmp_path / "config.json").write_text(json.dumps(dict(SD15_CONFIG, out_channels=4)))
    m = V.VAE_StableDiffusion(pretrained_path=str(tmp_path), device="cpu")     # the encoder still loads
    assert len(m.state_dict()) >= 108 and not m.has_decoder
    with pytest.raises(ValueError, match="out_channels"):
        m._decoder()


def test_checkpoint_routing_loads_a_complete_decoder(full):
    from nope_b200.unet import encoder_entries
    ckpt = {"encoder.encoder." + k: v for k, v in full.items()}
    ckpt["time_mlp.0.weight"] = torch.zeros(1)
    vae = V.VAE_StableDiffusion(device="cpu")
    got = encoder_entries(ckpt, vae)
    assert set(got) == set(full)
    assert vae.load_state_dict(got).has_decoder
    # a PoseConditional's state_dict() carries the decoder back under u_net.encoder.encoder.*
    assert {"encoder." + k for k in got} == set(vae.state_dict())


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("H,W", [(1, 1), (3, 5), (8, 8)])
def test_oracle_folded_upsample_equals_nearest_then_3x3(H, W):
    g = torch.Generator().manual_seed(H * 10 + W)
    x = torch.randn(2, 6, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(5, 6, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    ref = D.upsample(x, w, b)
    # by hand, borders included: output (Y, X) sums w[ky, kx] * up[Y + ky - 1, X + kx - 1], up[i] = x[i // 2]
    up = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
    hand = b[None, :, None, None].expand(2, 5, 2 * H, 2 * W).clone()
    for yy in range(2 * H):
        for xx in range(2 * W):
            for ky in range(3):
                for kx in range(3):
                    sy, sx = yy + ky - 1, xx + kx - 1
                    if 0 <= sy < 2 * H and 0 <= sx < 2 * W:
                        hand[:, :, yy, xx] += up[:, :, sy, sx] @ w[:, :, ky, kx].T
    assert torch.allclose(ref, hand, rtol=0, atol=1e-12)
    assert torch.allclose(D.upsample_folded(x, w, b), ref, rtol=0, atol=1e-12)


def test_oracle_decoder_flop_count():
    c = D.flops_per_image()
    # DESIGN.md section 17: 617.89 GFLOP of convolutions, 2.15 of q / k / v / proj_attn, 2.15 of attention products
    assert c == {"conv": 617892315136, "linear": 2147483648, "attention": 2147483648}
    assert round(sum(c.values()) / 1e9, 1) == 622.2


def test_oracle_decode_shapes_on_meta():
    sd = {k: torch.zeros(s, device="meta") for k, s in V.vae_decoder_param_shapes().items()}
    taps = {}
    y = D.decode(sd, torch.zeros(2, 4, 32, 32, device="meta"), taps=taps)
    assert y.shape == (2, 3, 256, 256)
    assert [tuple(taps[k].shape[1:]) for k in ("mid", "up0", "up1", "up2", "up3")] == \
        [(512, 32, 32), (512, 64, 64), (512, 128, 128), (256, 256, 256), (128, 256, 256)]


# ------------------------------------------------------------------ library
def test_vae_decoder_symbols_are_exported():
    from nope_b200 import _lib, build
    if not build.have_nvcc() and not os.path.exists(_lib.LIB_PATH):
        pytest.skip("neither nvcc nor a built library")
    lib = _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name in ("nope_vae_decoder_create", "nope_vae_decoder_load_tensor", "nope_vae_decoder_finalize",
                 "nope_vae_decoder_decode", "nope_vae_decoder_last_launch_count", "nope_vae_decoder_destroy"):
        assert name in _lib.SIGNATURES and hasattr(lib, name) and f" T {name}" in out, name
