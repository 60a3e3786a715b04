"""Seeded synthetic ("random-init") weights with the reference's state_dict schema
(SURVEY.md section 8b "Weights") -- input generation for the bench, the tools and the
tests; not part of any arithmetic.

No trained checkpoint ships with the reference, so benchmarks run on random-init weights of
the reference architecture and parity is pinned on the same seeded weights.  The recipe below does not need the reference tree: it
enumerates the keys/shapes that `UNet.state_dict()` and
`FeatureExtractor.state_dict()` produce
(reference: src/model/u_net/denoising_diffusion_pytorch/u_net.py:27-158,
src/model/encoder/template.py:24-45, src/model/encoder/resnet.py:93-133) and
fills each tensor from a torch CPU generator, which is platform independent.
`oracle/make_golden.py` loads the result into the reference's own modules with
strict=True, which pins the schema.

Distributions: conv/linear weights U(-b, b) with b = gain / sqrt(fan_in)
(PyTorch's default family), biases U(-b, b); norm weights 1 + 0.2 U(-1,1),
norm biases 0.2 U(-1,1) so affine-handling bugs are visible; BatchNorm running
mean 0.1 U(-1,1), running var 1 + 0.2 U(-1,1).
"""
from collections import OrderedDict
import math
import torch


def _resblock_shapes(prefix, cin, cout, cemb, with_mlp=True):
    s = OrderedDict()
    if with_mlp:
        s[f"{prefix}.mlp.1.weight"] = (cout, cemb)
        s[f"{prefix}.mlp.1.bias"] = (cout,)
    s[f"{prefix}.block1.proj.weight"] = (cout, cin, 3, 3)
    s[f"{prefix}.block1.proj.bias"] = (cout,)
    s[f"{prefix}.block1.norm.weight"] = (cout,)
    s[f"{prefix}.block1.norm.bias"] = (cout,)
    s[f"{prefix}.block2.proj.weight"] = (cout, cout, 3, 3)
    s[f"{prefix}.block2.proj.bias"] = (cout,)
    s[f"{prefix}.block2.norm.weight"] = (cout,)
    s[f"{prefix}.block2.norm.bias"] = (cout,)
    if cin != cout:
        s[f"{prefix}.res_conv.weight"] = (cout, cin, 1, 1)
        s[f"{prefix}.res_conv.bias"] = (cout,)
    return s


def _linattn_shapes(prefix, dim, hidden=128):
    # Residual(PreNorm(dim, LinearAttention(dim))): model_utils.py:393-418,226-234
    s = OrderedDict()
    s[f"{prefix}.fn.fn.to_qkv.weight"] = (hidden * 3, dim, 1, 1)
    s[f"{prefix}.fn.fn.to_out.0.weight"] = (dim, hidden, 1, 1)
    s[f"{prefix}.fn.fn.to_out.0.bias"] = (dim,)
    s[f"{prefix}.fn.fn.to_out.1.weight"] = (dim,)
    s[f"{prefix}.fn.fn.to_out.1.bias"] = (dim,)
    s[f"{prefix}.fn.norm.weight"] = (dim,)
    s[f"{prefix}.fn.norm.bias"] = (dim,)
    return s


def unet_param_shapes(u_net_dim=192, channels=8, rot_dim=6, dim_mults=(1, 2, 4, 8)):
    """Key -> shape for the default UNet, encoder keys excluded (u_net.py:27-158)."""
    cemb = u_net_dim * 4
    dims = [u_net_dim] + [u_net_dim * m for m in dim_mults]
    in_out = list(zip(dims[:-1], dims[1:]))
    s = OrderedDict()
    s["pose_mlp.0.weight"] = (cemb, rot_dim)
    s["pose_mlp.0.bias"] = (cemb,)
    s["init_conv.weight"] = (u_net_dim, channels, 3, 3)
    s["init_conv.bias"] = (u_net_dim,)
    for i, (din, dout) in enumerate(in_out):
        last = i == len(in_out) - 1
        s.update(_resblock_shapes(f"downs.{i}.0", din, din, cemb))
        s.update(_resblock_shapes(f"downs.{i}.1", din, din, cemb))
        s.update(_linattn_shapes(f"downs.{i}.2", din))
        if not last:
            s[f"downs.{i}.3.1.weight"] = (dout, din * 4, 1, 1)
            s[f"downs.{i}.3.1.bias"] = (dout,)
        else:
            s[f"downs.{i}.3.weight"] = (dout, din, 3, 3)
            s[f"downs.{i}.3.bias"] = (dout,)
    mid = dims[-1]
    # Residual(PreNorm(mid, Attention(mid))): model_utils.py:367-390
    s["mid_attn.fn.fn.to_qkv.weight"] = (384, mid, 1, 1)
    s["mid_attn.fn.fn.to_out.weight"] = (mid, 128, 1, 1)
    s["mid_attn.fn.fn.to_out.bias"] = (mid,)
    s["mid_attn.fn.norm.weight"] = (mid,)
    s["mid_attn.fn.norm.bias"] = (mid,)
    s.update(_resblock_shapes("mid_block1", mid, mid, cemb))
    s.update(_resblock_shapes("mid_block2", mid, mid, cemb))
    for i, (din, dout) in enumerate(reversed(in_out)):
        last = i == len(in_out) - 1
        s.update(_resblock_shapes(f"ups.{i}.0", dout + din, dout, cemb))
        s.update(_resblock_shapes(f"ups.{i}.1", dout + din, dout, cemb))
        s.update(_linattn_shapes(f"ups.{i}.2", dout))
        if not last:
            s[f"ups.{i}.3.1.weight"] = (din, dout, 3, 3)
            s[f"ups.{i}.3.1.bias"] = (din,)
        else:
            s[f"ups.{i}.3.weight"] = (din, dout, 3, 3)
            s[f"ups.{i}.3.bias"] = (din,)
    s.update(_resblock_shapes("final_res_block", u_net_dim * 2, u_net_dim, cemb))
    # final_conv.0 is a ResnetBlock built with the partial's time_emb_dim, so it
    # owns an (unused) mlp.1 as well (u_net.py:154-157; forward gets no emb).
    s.update(_resblock_shapes("final_conv.0", u_net_dim, u_net_dim, cemb))
    s["final_conv.1.weight"] = (channels, u_net_dim, 1, 1)
    s["final_conv.1.bias"] = (channels,)
    return s


def _bn_shapes(prefix, c):
    return OrderedDict([(f"{prefix}.weight", (c,)), (f"{prefix}.bias", (c,)),
                        (f"{prefix}.running_mean", (c,)), (f"{prefix}.running_var", (c,)),
                        (f"{prefix}.num_batches_tracked", ())])


def encoder_param_shapes(descriptor_size=8):
    """Key -> shape for FeatureExtractor.backbone/.projector (resnet.py:93-133,
    template.py:29-39).  The reference registers the same tensors a second time
    as encoder.{0,1}.* (template.py:40); `alias_encoder_keys` adds those."""
    s = OrderedDict()
    s["backbone.conv1.weight"] = (64, 3, 7, 7)
    s.update(_bn_shapes("backbone.bn1", 64))
    inplanes = 64
    for li, (planes, blocks, stride) in enumerate(
            [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 1)], start=1):
        for b in range(blocks):
            p = f"backbone.layer{li}.{b}"
            s[f"{p}.conv1.weight"] = (planes, inplanes, 1, 1)
            s.update(_bn_shapes(f"{p}.bn1", planes))
            s[f"{p}.conv2.weight"] = (planes, planes, 3, 3)
            s.update(_bn_shapes(f"{p}.bn2", planes))
            s[f"{p}.conv3.weight"] = (planes * 4, planes, 1, 1)
            s.update(_bn_shapes(f"{p}.bn3", planes * 4))
            if b == 0 and (stride != 1 or inplanes != planes * 4):
                s[f"{p}.downsample.0.weight"] = (planes * 4, inplanes, 1, 1)
                s.update(_bn_shapes(f"{p}.downsample.1", planes * 4))
            inplanes = planes * 4
    s["backbone.fc.weight"] = (1, 2048)   # resnet50(num_classes=1), unused
    s["backbone.fc.bias"] = (1,)
    s["projector.1.weight"] = (256, 2048, 1, 1)
    s["projector.3.weight"] = (descriptor_size, 256, 1, 1)
    return s


def _fill(name, shape, g):
    if len(shape) == 0:
        return torch.zeros((), dtype=torch.long)
    u = lambda: torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1
    leaf = name.rsplit(".", 1)[-1]
    is_norm = (".norm." in name or "to_out.1." in name or ".bn" in name
               or "downsample.1." in name)
    if leaf == "running_mean":
        return 0.1 * u()
    if leaf == "running_var":
        return 1.0 + 0.2 * u()
    if is_norm and len(shape) == 1:
        return (1.0 + 0.2 * u()) if leaf == "weight" else 0.2 * u()
    if leaf == "weight":
        fan_in = 1
        for d in shape[1:]:
            fan_in *= d
        gain = math.sqrt(3.0) if "backbone" in name or "projector" in name else 1.0
        return u() * (gain / math.sqrt(fan_in))
    # bias of conv / linear
    return u() * 0.1


def make_unet_state_dict(seed=0, u_net_dim=192, channels=8):
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    return OrderedDict((k, _fill(k, shp, g))
                       for k, shp in unet_param_shapes(u_net_dim, channels).items())


def make_encoder_state_dict(seed=0, descriptor_size=8):
    g = torch.Generator(device="cpu").manual_seed(2000 + seed)
    return OrderedDict((k, _fill(k, shp, g))
                       for k, shp in encoder_param_shapes(descriptor_size).items())


def alias_encoder_keys(enc_sd):
    """FeatureExtractor.state_dict() lists every tensor under backbone./projector.
    and again under encoder.0./encoder.1. (template.py:40)."""
    out = OrderedDict(enc_sd)
    for k, v in enc_sd.items():
        if k.startswith("backbone."):
            out["encoder.0." + k[len("backbone."):]] = v
        elif k.startswith("projector."):
            out["encoder.1." + k[len("projector."):]] = v
    return out


def make_full_state_dict(seed=0, u_net_dim=192, descriptor_size=8):
    """state_dict of reference `UNet` (u_net + 'encoder.'-prefixed encoder)."""
    sd = OrderedDict()
    enc = alias_encoder_keys(make_encoder_state_dict(seed, descriptor_size))
    for k, v in enc.items():
        sd["encoder." + k] = v
    sd.update(make_unet_state_dict(seed, u_net_dim, descriptor_size))
    return sd


def checksum(sd):
    """Order-sensitive fp64 checksum used to assert RNG determinism across boxes."""
    acc = 0.0
    for i, (k, v) in enumerate(sd.items()):
        if v.dtype.is_floating_point:
            acc += float(v.double().sum()) * (1 + (i % 7)) + float(v.double().abs().sum())
    return acc


# ---------------------------------------------------------------------------------------
# LDM variant: UNetModelPose (reference: src/model/u_net/ldm/adapt_openaimodel.py:14-125,
# src/model/u_net/ldm/openaimodel.py:428-760, src/model/u_net/ldm/attention.py:149-277;
# configs/model/vae_cin_ldm.yaml:2-31)
# ---------------------------------------------------------------------------------------
def _ldm_resblock_shapes(p, cin, cout, temb):
    s = OrderedDict()
    s[f"{p}.in_layers.0.weight"] = (cin,)
    s[f"{p}.in_layers.0.bias"] = (cin,)
    s[f"{p}.in_layers.2.weight"] = (cout, cin, 3, 3)
    s[f"{p}.in_layers.2.bias"] = (cout,)
    s[f"{p}.emb_layers.1.weight"] = (cout, temb)
    s[f"{p}.emb_layers.1.bias"] = (cout,)
    s[f"{p}.out_layers.0.weight"] = (cout,)
    s[f"{p}.out_layers.0.bias"] = (cout,)
    s[f"{p}.out_layers.3.weight"] = (cout, cout, 3, 3)
    s[f"{p}.out_layers.3.bias"] = (cout,)
    if cin != cout:
        s[f"{p}.skip_connection.weight"] = (cout, cin, 1, 1)
        s[f"{p}.skip_connection.bias"] = (cout,)
    return s


def _ldm_transformer_shapes(p, c, ctx):
    s = OrderedDict()
    s[f"{p}.norm.weight"] = (c,)
    s[f"{p}.norm.bias"] = (c,)
    s[f"{p}.proj_in.weight"] = (c, c, 1, 1)
    s[f"{p}.proj_in.bias"] = (c,)
    t = f"{p}.transformer_blocks.0"
    for a, kdim in (("attn1", c), ("attn2", ctx)):
        s[f"{t}.{a}.to_q.weight"] = (c, c)
        s[f"{t}.{a}.to_k.weight"] = (c, kdim)
        s[f"{t}.{a}.to_v.weight"] = (c, kdim)
        s[f"{t}.{a}.to_out.0.weight"] = (c, c)
        s[f"{t}.{a}.to_out.0.bias"] = (c,)
    s[f"{t}.ff.net.0.proj.weight"] = (8 * c, c)
    s[f"{t}.ff.net.0.proj.bias"] = (8 * c,)
    s[f"{t}.ff.net.2.weight"] = (c, 4 * c)
    s[f"{t}.ff.net.2.bias"] = (c,)
    for n in ("norm1", "norm2", "norm3"):
        s[f"{t}.{n}.weight"] = (c,)
        s[f"{t}.{n}.bias"] = (c,)
    s[f"{p}.proj_out.weight"] = (c, c, 1, 1)
    s[f"{p}.proj_out.bias"] = (c,)
    return s


def ldm_block_plan(model_channels=256, channel_mult=(1, 2, 4), num_res_blocks=2):
    """The module list UNetModel.__init__ builds (openaimodel.py:543-719) for attention at every
    level (vae_cin_ldm.yaml:8-16), as plain tuples:
      input:  ("conv"|"res"|"down", cin, cout)   -- "res" is ResBlock + SpatialTransformer
      middle: [("res", ch, ch), ("st", ch), ("res", ch, ch)]
      output: ("res", cin_total, cout, skip_ch, upsample)"""
    mc = model_channels
    inp = [("conv", None, mc)]
    chans = [mc]
    ch = mc
    for level, mult in enumerate(channel_mult):
        for _ in range(num_res_blocks):
            inp.append(("res", ch, mult * mc))
            ch = mult * mc
            chans.append(ch)
        if level != len(channel_mult) - 1:
            inp.append(("down", ch, ch))
            chans.append(ch)
    mid_ch = ch
    out = []
    for level, mult in list(enumerate(channel_mult))[::-1]:
        for i in range(num_res_blocks + 1):
            ich = chans.pop()
            out.append(("res", ch + ich, mc * mult, ich, bool(level and i == num_res_blocks)))
            ch = mc * mult
    return inp, mid_ch, out


def ldm_param_shapes(model_channels=256, channel_mult=(1, 2, 4), num_res_blocks=2, in_channels=4,
                     out_channels=4, context_dim=512, rot_dim=6):
    """Key -> shape of UNetModelPose.state_dict() without the (stubbed) encoder."""
    mc = model_channels
    temb = 4 * mc
    inp, mid_ch, out = ldm_block_plan(mc, channel_mult, num_res_blocks)
    s = OrderedDict()
    s["time_embed.0.weight"] = (temb, mc)      # present in the state_dict, unused by forward
    s["time_embed.0.bias"] = (temb,)           # (adapt_openaimodel.py:139-146: emb = zeros)
    s["time_embed.2.weight"] = (temb, temb)
    s["time_embed.2.bias"] = (temb,)
    for i, b in enumerate(inp):
        p = f"input_blocks.{i}"
        if b[0] == "conv":
            s[f"{p}.0.weight"] = (mc, in_channels, 3, 3)
            s[f"{p}.0.bias"] = (mc,)
        elif b[0] == "res":
            s.update(_ldm_resblock_shapes(f"{p}.0", b[1], b[2], temb))
            s.update(_ldm_transformer_shapes(f"{p}.1", b[2], context_dim))
        else:
            s[f"{p}.0.op.weight"] = (b[2], b[1], 3, 3)
            s[f"{p}.0.op.bias"] = (b[2],)
    s.update(_ldm_resblock_shapes("middle_block.0", mid_ch, mid_ch, temb))
    s.update(_ldm_transformer_shapes("middle_block.1", mid_ch, context_dim))
    s.update(_ldm_resblock_shapes("middle_block.2", mid_ch, mid_ch, temb))
    for i, b in enumerate(out):
        p = f"output_blocks.{i}"
        s.update(_ldm_resblock_shapes(f"{p}.0", b[1], b[2], temb))
        s.update(_ldm_transformer_shapes(f"{p}.1", b[2], context_dim))
        if b[4]:
            s[f"{p}.2.conv.weight"] = (b[2], b[2], 3, 3)
            s[f"{p}.2.conv.bias"] = (b[2],)
    s["out.0.weight"] = (mc,)
    s["out.0.bias"] = (mc,)
    s["out.2.weight"] = (out_channels, mc, 3, 3)
    s["out.2.bias"] = (out_channels,)
    s["pose_mlp.0.weight"] = (context_dim, rot_dim)
    s["pose_mlp.0.bias"] = (context_dim,)
    return s


def _fill_ldm(name, shape, g):
    u = lambda: torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1
    leaf = name.rsplit(".", 1)[-1]
    if len(shape) == 1 and any(t in name for t in (".in_layers.0.", ".out_layers.0.", ".norm.",
                                                    ".norm1.", ".norm2.", ".norm3.", "out.0.")):
        return (1.0 + 0.2 * u()) if leaf == "weight" else 0.2 * u()
    if leaf == "weight":
        fan_in = 1
        for d in shape[1:]:
            fan_in *= d
        # unit-variance outputs (the reference zero-initialises out_layers.3 / proj_out / out.2,
        # openaimodel.py:241-245,722-726 + attention.py:243-245, which would make the whole net a
        # no-op: every layer gets live weights here); q/k a little hotter so the softmax over
        # tokens is far from uniform
        gain = math.sqrt(3.0) * (1.5 if (".to_q." in name or ".to_k." in name) else 1.0)
        if ".proj_out." in name or ".out_layers.3." in name or ".ff.net.2." in name or ".to_out." in name:
            gain *= 0.5     # residual branches: keep the residual stream's growth moderate
        return u() * (gain / math.sqrt(fan_in))
    return u() * 0.1


def make_ldm_state_dict(seed=0, model_channels=256, channel_mult=(1, 2, 4), context_dim=512):
    g = torch.Generator(device="cpu").manual_seed(3000 + seed)
    return OrderedDict((k, _fill_ldm(k, shp, g)) for k, shp in
                       ldm_param_shapes(model_channels, channel_mult, context_dim=context_dim).items())


def ldm_flops_per_hyp(model_channels=256, channel_mult=(1, 2, 4), num_res_blocks=2, latent=32,
                      in_channels=4):
    """Algorithmic FLOPs of one UNetModelPose.forward (2 x multiply-adds): convolutions / linear
    layers as 2*M*N*K and the self-attention contractions (QK^T and PV); the one-token
    cross-attention and the unused time embedding are not counted."""
    inp, mid_ch, out = ldm_block_plan(model_channels, channel_mult, num_res_blocks)
    gemm = 0.0
    attn = 0.0

    def res(cin, cout, hw):
        f = 2.0 * hw * cout * cin * 9 + 2.0 * hw * cout * cout * 9
        if cin != cout:
            f += 2.0 * hw * cout * cin
        return f

    def st(c, hw):
        lin = 2.0 * hw * c * c * (1 + 3 + 1 + 1) + 2.0 * hw * c * 8 * c + 2.0 * hw * 4 * c * c
        return lin, 4.0 * hw * hw * c

    S = latent
    for b in inp:
        if b[0] == "conv":
            gemm += 2.0 * S * S * b[2] * in_channels * 9
        elif b[0] == "res":
            gemm += res(b[1], b[2], S * S)
            l, a = st(b[2], S * S)
            gemm += l
            attn += a
        else:
            S //= 2
            gemm += 2.0 * S * S * b[2] * b[1] * 9
    gemm += 2 * res(mid_ch, mid_ch, S * S)
    l, a = st(mid_ch, S * S)
    gemm += l
    attn += a
    for b in out:
        gemm += res(b[1], b[2], S * S)
        l, a = st(b[2], S * S)
        gemm += l
        attn += a
        if b[4]:
            S *= 2
            gemm += 2.0 * S * S * b[2] * b[2] * 9
    gemm += 2.0 * S * S * in_channels * model_channels * 9
    return {"gemm": gemm, "attention": attn, "total": gemm + attn}


def make_vae_state_dict(seed=0, attention="legacy", decoder=False):
    """Seeded AutoencoderKL encoder state_dict (nope_b200.vae.vae_param_shapes, 108 tensors, 34.16 M parameters):
    conv / linear weights and biases U(-1, 1) / sqrt(fan_in) (torch's default init), GroupNorm weights
    1 + 0.2 U(-1, 1) and biases 0.2 U(-1, 1), so activations stay O(1) through the 22 GroupNorms.
    attention="legacy" names the mid-block projections query / key / value / proj_attn (diffusers 0.14),
    "new" to_q / to_k / to_v / to_out.0; both hold the same tensors.  decoder=True appends the 140 decoder tensors
    (nope_b200.vae.vae_decoder_param_shapes, 49.49 M parameters) with the same rules from a generator of their own,
    so the encoder tensors are those of decoder=False."""
    from .vae import vae_decoder_param_shapes, vae_param_shapes
    if attention not in ("legacy", "new"):
        raise ValueError("attention must be 'legacy' or 'new'")
    rename = {"query.": "to_q.", "key.": "to_k.", "value.": "to_v.", "proj_attn.": "to_out.0."}
    sd = OrderedDict()
    parts = [(vae_param_shapes(), 5000 + seed, "encoder.mid_block.attentions.0.")]
    if decoder:
        parts.append((vae_decoder_param_shapes(), 6000 + seed, "decoder.mid_block.attentions.0."))
    for shapes, gseed, attn in parts:
        g = torch.Generator(device="cpu").manual_seed(gseed)
        fan = {}
        for k, shape in shapes.items():
            u = torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1
            p, leaf = k.rsplit(".", 1)
            if "norm" in p:
                t = 1.0 + 0.2 * u if leaf == "weight" else 0.2 * u
            else:
                if leaf == "weight":
                    fan[p] = math.prod(shape[1:])
                t = u / math.sqrt(fan[p])
            if attention == "new" and k.startswith(attn):
                for a, b in rename.items():
                    if k[len(attn):].startswith(a):
                        k = attn + b + k[len(attn) + len(a):]
            sd[k] = t
    return sd
