"""TEST INFRASTRUCTURE ONLY -- functional float64 restatement of the Stable Diffusion VAE encoder,
`AutoencoderKL.encode(x).latent_dist.mode() * 0.18215` of the SD v1 configuration (DESIGN.md section 16,
the specification nope_b200/csrc/vae.cuh implements), over a plain state_dict with diffusers' key names.
diffusers is not available here, so this module is written from the specification, not checked against
diffusers' code: DESIGN.md section 16 lists the points where the two could differ.

Runs on CPU or on a CUDA device, in float64 unless told otherwise.  Only tests/ and tools/ may import it.
"""
import torch
import torch.nn.functional as F

ATTN = "encoder.mid_block.attentions.0."
_NEW_NAMES = {"to_q.": "query.", "to_k.": "key.", "to_v.": "value.", "to_out.0.": "proj_attn."}
SCALE = 0.18215


def canonical(sd, device="cpu", dtype=torch.float64):
    """Either attention naming -> the 0.14-era names; decoder.* / post_quant_conv.* dropped."""
    out = {}
    for k, v in sd.items():
        if k.startswith("decoder.") or k.startswith("post_quant_conv."):
            continue
        if k.startswith(ATTN):
            for a, b in _NEW_NAMES.items():
                if k[len(ATTN):].startswith(a):
                    k = ATTN + b + k[len(ATTN) + len(a):]
        out[k] = v.to(device=device, dtype=dtype)
    return out


def group_norm(x, sd, p, eps=1e-6):
    return F.group_norm(x, 32, sd[p + ".weight"], sd[p + ".bias"], eps)


def resnet(x, sd, p):
    """ResnetBlock2D (no time embedding, output_scale_factor 1): shortcut(x) + conv2(SiLU(GN2(conv1(SiLU(GN1(x))))))."""
    h = F.conv2d(F.silu(group_norm(x, sd, p + ".norm1")), sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], padding=1)
    h = F.conv2d(F.silu(group_norm(h, sd, p + ".norm2")), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"], padding=1)
    if p + ".conv_shortcut.weight" in sd:
        x = F.conv2d(x, sd[p + ".conv_shortcut.weight"], sd[p + ".conv_shortcut.bias"])
    return x + h


def downsample(x, w, b):
    """Downsample2D(padding=0): zero pad one row at the bottom and one column at the right, 3x3 stride 2."""
    return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)


def softmax(s):
    e = torch.exp(s - s.max(dim=-1, keepdim=True).values)
    return e / e.sum(dim=-1, keepdim=True)


def attention(x, sd, p=ATTN):
    """One-head self-attention over the H*W tokens: x + proj_attn(softmax(q k^T / sqrt(C)) v), q, k, v = Linear(GN(x))."""
    B, Cc, H, W = x.shape
    t = group_norm(x, sd, p + "group_norm").reshape(B, Cc, H * W).transpose(1, 2)
    q = F.linear(t, sd[p + "query.weight"], sd[p + "query.bias"])
    k = F.linear(t, sd[p + "key.weight"], sd[p + "key.bias"])
    v = F.linear(t, sd[p + "value.weight"], sd[p + "value.bias"])
    o = torch.matmul(softmax(torch.matmul(q, k.transpose(1, 2)) / Cc ** 0.5), v)
    o = F.linear(o, sd[p + "proj_attn.weight"], sd[p + "proj_attn.bias"])
    return x + o.transpose(1, 2).reshape(B, Cc, H, W)


@torch.no_grad()
def encode(sd, x, taps=None, dtype=torch.float64):
    """x [B, 3, 256, 256] -> latent [B, 4, 32, 32] (dtype).  taps, if a dict, receives the activations after
    each down block ("down0" .. "down3") and after the mid block ("mid"), and (input, output) of every module the
    engine runs on its own (nope_vae_run_block) under its name: "encoder.conv_in",
    "encoder.down_blocks.<i>.resnets.<j>", "encoder.down_blocks.<i>.downsamplers.0", "encoder.mid_block.resnets.<j>",
    "encoder.mid_block.attentions.0" and "encoder.conv_out" (conv_norm_out + SiLU + conv_out + quant_conv mean x
    0.18215, whose output is the latent)."""
    sd = canonical(sd, x.device, dtype)
    x = x.to(dtype)

    def module(name, fn, h):
        out = fn(h)
        if taps is not None:
            taps[name] = (h, out)
        return out

    h = module("encoder.conv_in", lambda t: F.conv2d(t, sd["encoder.conv_in.weight"], sd["encoder.conv_in.bias"],
                                                     padding=1), x)
    for i in range(4):
        for j in range(2):
            p = f"encoder.down_blocks.{i}.resnets.{j}"
            h = module(p, lambda t: resnet(t, sd, p), h)
        if i < 3:
            p = f"encoder.down_blocks.{i}.downsamplers.0"
            h = module(p, lambda t: downsample(t, sd[p + ".conv.weight"], sd[p + ".conv.bias"]), h)
        if taps is not None:
            taps[f"down{i}"] = h
    h = module("encoder.mid_block.resnets.0", lambda t: resnet(t, sd, "encoder.mid_block.resnets.0"), h)
    h = module("encoder.mid_block.attentions.0", lambda t: attention(t, sd), h)
    h = module("encoder.mid_block.resnets.1", lambda t: resnet(t, sd, "encoder.mid_block.resnets.1"), h)
    if taps is not None:
        taps["mid"] = h
    return module("encoder.conv_out", lambda t: conv_out(t, sd), h)


def conv_out(h, sd):
    """conv_norm_out + SiLU, conv_out, quant_conv, the mean's four channels x 0.18215"""
    h = F.silu(group_norm(h, sd, "encoder.conv_norm_out"))
    h = F.conv2d(h, sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], padding=1)
    h = F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])
    return h[:, :4] * SCALE


def flops_per_image():
    """2 x the multiply-adds of every convolution, linear and attention product of one 256 x 256 image, counted by
    wrapping the oracle's F.conv2d / F.linear / torch.matmul during an encode on meta tensors."""
    from nope_b200.vae import vae_param_shapes
    counts = {"conv": 0, "linear": 0, "attention": 0}
    real_conv, real_linear, real_matmul = F.conv2d, F.linear, torch.matmul

    def conv(x, w, b=None, stride=1, padding=0, **kw):
        y = real_conv(x, w, b, stride=stride, padding=padding)
        counts["conv"] += 2 * y.numel() * w.shape[1] * w.shape[2] * w.shape[3]
        return y

    def linear(x, w, b=None):
        y = real_linear(x, w, b)
        counts["linear"] += 2 * y.numel() * w.shape[1]
        return y

    def matmul(a, b):
        y = real_matmul(a, b)
        counts["attention"] += 2 * y.numel() * a.shape[-1]
        return y

    sd = {k: torch.zeros(s, device="meta") for k, s in vae_param_shapes().items()}
    F.conv2d, F.linear, torch.matmul = conv, linear, matmul
    try:
        encode(sd, torch.zeros(1, 3, 256, 256, device="meta"))
    finally:
        F.conv2d, F.linear, torch.matmul = real_conv, real_linear, real_matmul
    return counts
