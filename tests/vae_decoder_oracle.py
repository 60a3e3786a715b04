"""TEST INFRASTRUCTURE ONLY -- functional float64 restatement of the Stable Diffusion VAE decoder,
`AutoencoderKL.decode(z / 0.18215).sample` of the SD v1 configuration (DESIGN.md section 17, the specification
the decoder half of nope_b200/csrc/vae.cuh implements), over a plain state_dict with diffusers' key names.  It
reuses the encoder oracle's ResnetBlock2D, attention and GroupNorm (oracle/vae_oracle.py), which the decoder's
blocks share.  diffusers is not available here, so this is written from the specification, not checked against
diffusers' code: DESIGN.md section 17 lists the points where the two could differ.

Runs on CPU or on a CUDA device, in float64 unless told otherwise.  Only tests/ and tools/ import it.
"""
import torch
import torch.nn.functional as F

from oracle import vae_oracle as E

ATTN = "decoder.mid_block.attentions.0."
CHANNELS = (512, 512, 256, 128)
# parity p -> source offset index a (offset p - 1 + a) -> the taps k of a 3x3 kernel that land on it after a
# nearest x2 upsample: output 2Y + p, tap k reads source row Y + floor((p + k - 1) / 2)
_FOLD = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}


def canonical(sd, device="cpu", dtype=torch.float64):
    """The decoder.* / post_quant_conv.* entries, either attention naming -> the 0.14-era names."""
    out = {}
    for k, v in sd.items():
        if not (k.startswith("decoder.") or k.startswith("post_quant_conv.")):
            continue
        if k.startswith(ATTN):
            for a, b in E._NEW_NAMES.items():
                if k[len(ATTN):].startswith(a):
                    k = ATTN + b + k[len(ATTN) + len(a):]
        out[k] = v.to(device=device, dtype=dtype)
    return out


def upsample(x, w, b):
    """Upsample2D: nearest x2, then a 3x3 pad-1 convolution."""
    return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, b, padding=1)


def fold_upsample_weight(w):
    """[Co, Ci, 3, 3] -> [4, Co, Ci, 2, 2]: the 2x2 kernel of each output parity (py, px) = index 2 py + px, whose
    tap (a, b) reads the source at offset (py - 1 + a, px - 1 + b)."""
    out = w.new_zeros((4,) + tuple(w.shape[:2]) + (2, 2))
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    for ky in _FOLD[py][a]:
                        for kx in _FOLD[px][b]:
                            out[2 * py + px, :, :, a, b] += w[:, :, ky, kx]
    return out


def upsample_folded(x, w, b):
    """upsample() as four 2x2 convolutions over the source, one per output parity, zero padded by one."""
    B, _, H, W = x.shape
    wf = fold_upsample_weight(w)
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros((B, w.shape[0], 2 * H, 2 * W))
    for py in range(2):
        for px in range(2):
            out[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], wf[2 * py + px], b)
    return out


@torch.no_grad()
def decode(sd, z, taps=None, dtype=torch.float64):
    """z [B, 4, 32, 32] -> image [B, 3, 256, 256] (dtype), not clamped.  taps, if a dict, receives the activations
    after the mid block ("mid") and after each up block ("up0" .. "up3"), and (input, output) of every module the
    engine runs on its own (nope_vae_decoder_run_block) under its name: "decoder.conv_in" (post_quant_conv with
    1 / 0.18215, then conv_in), "decoder.mid_block.resnets.<j>", "decoder.mid_block.attentions.0",
    "decoder.up_blocks.<i>.resnets.<j>", "decoder.up_blocks.<i>.upsamplers.0" and "decoder.conv_out"
    (conv_norm_out + SiLU + conv_out, whose output is the image)."""
    sd = canonical(sd, z.device, dtype)

    def module(name, fn, h):
        out = fn(h)
        if taps is not None:
            taps[name] = (h, out)
        return out

    def conv_in(t):
        t = F.conv2d(t / E.SCALE, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
        return F.conv2d(t, sd["decoder.conv_in.weight"], sd["decoder.conv_in.bias"], padding=1)

    def conv_out(t):
        t = F.silu(E.group_norm(t, sd, "decoder.conv_norm_out"))
        return F.conv2d(t, sd["decoder.conv_out.weight"], sd["decoder.conv_out.bias"], padding=1)

    h = module("decoder.conv_in", conv_in, z.to(dtype))
    h = module("decoder.mid_block.resnets.0", lambda t: E.resnet(t, sd, "decoder.mid_block.resnets.0"), h)
    h = module("decoder.mid_block.attentions.0", lambda t: E.attention(t, sd, ATTN), h)
    h = module("decoder.mid_block.resnets.1", lambda t: E.resnet(t, sd, "decoder.mid_block.resnets.1"), h)
    if taps is not None:
        taps["mid"] = h
    for i in range(4):
        for j in range(3):
            p = f"decoder.up_blocks.{i}.resnets.{j}"
            h = module(p, lambda t: E.resnet(t, sd, p), h)
        if i < 3:
            p = f"decoder.up_blocks.{i}.upsamplers.0"
            h = module(p, lambda t: upsample(t, sd[p + ".conv.weight"], sd[p + ".conv.bias"]), h)
        if taps is not None:
            taps[f"up{i}"] = h
    return module("decoder.conv_out", conv_out, h)


def flops_per_image():
    """2 x the multiply-adds of every convolution, linear and attention product of one 32 x 32 latent's decode,
    counted by wrapping F.conv2d / F.linear / torch.matmul during a decode on meta tensors (as
    vae_oracle.flops_per_image does for the encoder)."""
    from nope_b200.vae import vae_decoder_param_shapes
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

    sd = {k: torch.zeros(s, device="meta") for k, s in vae_decoder_param_shapes().items()}
    F.conv2d, F.linear, torch.matmul = conv, linear, matmul
    try:
        decode(sd, torch.zeros(1, 4, 32, 32, device="meta"))
    finally:
        F.conv2d, F.linear, torch.matmul = real_conv, real_linear, real_matmul
    return counts
