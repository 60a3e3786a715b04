"""CPU: the SD VAE encoder's host side (nope_b200.vae): config parsing, the AutoencoderKL key mapping and the seeded
recipe's schema, checkpoint routing to the encoder in both UNets, the float64 oracle's building blocks against
textbook restatements, the FLOP count DESIGN.md section 16 records, and the new ABI symbols."""
import copy
import json
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from _util import SD15_CONFIG
from nope_b200 import vae as V

OTHER_VALUES = {
    "in_channels": [1, 4], "latent_channels": [8, 16], "block_out_channels": [[128, 256, 512], [64, 128, 256, 256]],
    "down_block_types": [["DownEncoderBlock2D"] * 3, ["AttnDownEncoderBlock2D"] * 4], "layers_per_block": [1, 3],
    "norm_num_groups": [16, 8], "act_fn": ["relu", "gelu"], "double_z": [False],
}


@pytest.fixture(scope="module")
def sd():
    from nope_b200.synth_weights import make_vae_state_dict
    return make_vae_state_dict(seed=0)


def test_config_accepted_and_every_other_value_refused():
    V.check_config(SD15_CONFIG)
    V.check_config(dict(SD15_CONFIG, double_z=True, scaling_factor=0.18215))
    for k, values in OTHER_VALUES.items():
        for v in values:
            with pytest.raises(ValueError, match=k):
                V.check_config(dict(SD15_CONFIG, **{k: v}))
    for k in ("block_out_channels", "layers_per_block", "down_block_types"):   # diffusers' defaults differ
        cfg = dict(SD15_CONFIG)
        del cfg[k]
        with pytest.raises(ValueError, match=k):
            V.check_config(cfg)


def test_schema_counts(sd):
    # 108 encoder tensors, 34 163 664 parameters: conv_in 2, 8 down-block resnets 64 + 2 shortcuts 4, 3 downsamplers
    # 6, 2 mid resnets 16, attention 10, conv_norm_out 2, conv_out 2, quant_conv 2
    assert list(sd) == list(V.vae_param_shapes())
    assert len(sd) == 108
    assert sum(v.numel() for v in sd.values()) == 34163664
    assert all(tuple(v.shape) == s for v, s in zip(sd.values(), V.vae_param_shapes().values()))


def test_both_attention_namings_load_the_same_tensors(sd):
    from nope_b200.synth_weights import make_vae_state_dict
    new = make_vae_state_dict(seed=0, attention="new")
    assert "encoder.mid_block.attentions.0.to_out.0.weight" in new and "encoder.mid_block.attentions.0.query.bias" \
        not in new
    a, b = V.map_state_dict(sd), V.map_state_dict(new)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_decoder_entries_are_ignored_and_bad_entries_raise(sd):
    full = dict(sd)
    full["decoder.conv_in.weight"] = torch.zeros(512, 4, 3, 3)
    full["post_quant_conv.weight"] = torch.zeros(4, 4, 1, 1)
    m = V.map_state_dict(full)
    assert len(m) == 108 and all(torch.equal(m[k], sd[k]) for k in m)
    missing = dict(sd)
    del missing["encoder.down_blocks.1.resnets.0.conv_shortcut.bias"]
    with pytest.raises(KeyError, match="missing"):
        V.map_state_dict(missing)
    wrong = dict(sd)
    wrong["encoder.mid_block.attentions.0.key.weight"] = torch.zeros(512, 512, 1, 1)
    with pytest.raises(ValueError, match="size mismatch"):
        V.map_state_dict(wrong)
    with pytest.raises(KeyError, match="unexpected"):
        V.map_state_dict(dict(sd, **{"encoder.mid_block.attentions.0.proj.weight": torch.zeros(1)}))


def test_constructor_and_pretrained_directory(sd, tmp_path):
    with pytest.raises(ValueError):
        V.VAE_StableDiffusion(using_KL=True)
    with pytest.raises(ValueError):
        V.VAE_StableDiffusion(latent_dim=8)
    (tmp_path / "config.json").write_text(json.dumps(SD15_CONFIG))
    torch.save(dict(sd, **{"decoder.conv_out.bias": torch.zeros(3)}), tmp_path / "diffusion_pytorch_model.bin")
    m = V.VAE_StableDiffusion(pretrained_path=str(tmp_path), name="VAE", device="cpu")
    assert (m.latent_dim, m.name, m.using_KL, m.encode_mode) == (4, "VAE", False, "mode")
    st = m.state_dict()
    assert len(st) == 108 and torch.equal(st["encoder.quant_conv.weight"], sd["quant_conv.weight"])
    with pytest.raises(Exception):                      # no CPU path
        m.encode_image(torch.zeros(1, 3, 256, 256))
    (tmp_path / "config.json").write_text(json.dumps(dict(SD15_CONFIG, latent_channels=16)))
    with pytest.raises(ValueError):
        V.VAE_StableDiffusion(pretrained_path=str(tmp_path), device="cpu")


def test_checkpoint_routing(sd, seeded_state_dict):
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.unet import encoder_entries
    vae = V.VAE_StableDiffusion(device="cpu")
    ckpt = {"encoder.encoder." + k: v for k, v in sd.items()}       # u_net.encoder.encoder.* without "u_net."
    ckpt["encoder.encoder.decoder.conv_in.bias"] = torch.zeros(512)
    ckpt["time_mlp.0.weight"] = torch.zeros(1)
    got = encoder_entries(ckpt, vae)
    assert set(got) == set(sd) | {"decoder.conv_in.bias"}
    assert len(V.map_state_dict(got)) == 108
    # the template encoder: exactly the backbone / projector entries, as before
    fe = FeatureExtractor()
    got = encoder_entries(seeded_state_dict, fe)
    want = {k[len("encoder."):]: v for k, v in seeded_state_dict.items()
            if k.startswith("encoder.backbone.") or k.startswith("encoder.projector.")}
    assert set(got) == set(want) and all(got[k] is want[k] for k in want)
    assert encoder_entries(ckpt, fe) == {}


# ------------------------------------------------------------------ oracle building blocks
def test_oracle_downsample_is_stride_2_with_bottom_right_padding():
    from oracle import vae_oracle
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 7, 8, generator=g, dtype=torch.float64)
    w = torch.randn(5, 3, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    y = vae_oracle.downsample(x, w, b)
    Ho, Wo = 3, 4                                         # floor((7 + 1 - 3) / 2) + 1, floor((8 + 1 - 3) / 2) + 1
    ref = torch.zeros(2, 5, Ho, Wo, dtype=torch.float64)
    for yy in range(Ho):
        for xx in range(Wo):
            acc = b.clone()[None].expand(2, -1).clone()
            for ky in range(3):
                for kx in range(3):
                    sy, sx = 2 * yy + ky, 2 * xx + kx     # taps at 2y, 2y + 1, 2y + 2; zero past the bottom / right
                    if sy < 7 and sx < 8:
                        acc += x[:, :, sy, sx] @ w[:, :, ky, kx].T
            ref[:, :, yy, xx] = acc
    assert y.shape == ref.shape and torch.allclose(y, ref, rtol=0, atol=1e-12)


def test_oracle_attention_is_textbook_single_head():
    from oracle import vae_oracle
    g = torch.Generator().manual_seed(2)
    C, H = 64, 4
    x = torch.randn(2, C, H, H, generator=g, dtype=torch.float64)
    p = "a."
    sd = {p + "group_norm.weight": 1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64),
          p + "group_norm.bias": 0.1 * torch.randn(C, generator=g, dtype=torch.float64)}
    for n in ("query", "key", "value", "proj_attn"):
        sd[p + n + ".weight"] = torch.randn(C, C, generator=g, dtype=torch.float64) / 8
        sd[p + n + ".bias"] = torch.randn(C, generator=g, dtype=torch.float64) / 8
    y = vae_oracle.attention(x, sd, p)
    gn = torch.nn.GroupNorm(32, C, eps=1e-6).double()
    gn.weight.data, gn.bias.data = sd[p + "group_norm.weight"], sd[p + "group_norm.bias"]
    for b in range(2):
        t = gn(x[b:b + 1])[0].reshape(C, H * H).T                       # tokens x channels
        q, k, v = (t @ sd[p + n + ".weight"].T + sd[p + n + ".bias"] for n in ("query", "key", "value"))
        a = torch.softmax(q @ k.T / C ** 0.5, dim=-1)
        o = (a @ v) @ sd[p + "proj_attn.weight"].T + sd[p + "proj_attn.bias"]
        assert torch.allclose(y[b], x[b] + o.T.reshape(C, H, H), rtol=0, atol=1e-12)


def test_oracle_four_channel_group_norm_is_torch_group_norm():
    from oracle import vae_oracle
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 128, 8, 8, generator=g, dtype=torch.float64) * 3 + 1
    sd = {"n.weight": 1 + 0.2 * torch.randn(128, generator=g, dtype=torch.float64),
          "n.bias": 0.2 * torch.randn(128, generator=g, dtype=torch.float64)}
    gn = torch.nn.GroupNorm(32, 128, eps=1e-6).double()
    gn.weight.data, gn.bias.data = sd["n.weight"], sd["n.bias"]
    assert torch.allclose(vae_oracle.group_norm(x, sd, "n"), gn(x), rtol=0, atol=1e-12)
    xm = x.reshape(2, 32, 4, 8, 8)                                      # 4 channels per group, by hand
    ref = (xm - xm.mean((2, 3, 4), keepdim=True)) / torch.sqrt(xm.var((2, 3, 4), unbiased=False, keepdim=True) + 1e-6)
    ref = ref.reshape(2, 128, 8, 8) * sd["n.weight"][:, None, None] + sd["n.bias"][:, None, None]
    assert torch.allclose(vae_oracle.group_norm(x, sd, "n"), ref, rtol=0, atol=1e-12)


def test_oracle_flop_count():
    from oracle import vae_oracle
    c = vae_oracle.flops_per_image()
    # DESIGN.md section 16: 268.43 GFLOP of convolutions, 2.15 of q / k / v / proj_attn, 2.15 of attention products
    assert c == {"conv": 268427198464, "linear": 2147483648, "attention": 2147483648}


def test_oracle_takes_either_attention_naming(sd):
    from nope_b200.synth_weights import make_vae_state_dict
    from oracle import vae_oracle
    new = make_vae_state_dict(seed=0, attention="new")
    a, b = vae_oracle.canonical(sd), vae_oracle.canonical(new)
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)


# ------------------------------------------------------------------ library
def test_vae_symbols_are_exported():
    from nope_b200 import _lib, build
    if not build.have_nvcc() and not os.path.exists(_lib.LIB_PATH):
        pytest.skip("neither nvcc nor a built library")
    lib = _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name in ("nope_vae_create", "nope_vae_load_tensor", "nope_vae_finalize", "nope_vae_encode",
                 "nope_vae_encode_inplane", "nope_vae_encode_rotated", "nope_vae_last_launch_count",
                 "nope_vae_destroy"):
        assert name in _lib.SIGNATURES and hasattr(lib, name) and f" T {name}" in out, name
