import contextlib
import json
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "gpurun_out", "parity_log.jsonl")


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_rel(a, b):
    """max |a-b| / max|b|"""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def log(name, **vals):
    try:
        os.makedirs(os.path.dirname(LOG), exist_ok=True)
        with open(LOG, "a") as f:
            f.write(json.dumps({"test": name, **vals}) + "\n")
    except OSError:
        pass
    print(name, vals)


def h(t):
    """round to fp16 and back: the precision the kernels store activations / weights in"""
    return t.half().float()


def pick_bn(cout, ldm=False):
    """N-tile width the engines choose for `cout` output channels (pick_bn in csrc/conv_tc.cuh; the LDM engine
    takes 256-wide tiles wherever they divide)"""
    if ldm and cout % 256 == 0:
        return 256
    return next(bn for bn in (192, 128, 64) if cout % bn == 0)


def pair_tiles(n, H, W, cout, bn, n_par=1):
    """Tile pairs of one conv_tc2_kernel launch: ceil(m_tiles / 2) * n_tiles, with m_tiles over the 128-row tiles of
    the n*H*W output pixels (source pixels for the folded upsample, n_par = 4 parities).  Each 2-CTA cluster walks
    tile pairs cluster, cluster + clusters, ...: a launch runs pair_tiles / clusters rounds."""
    hw = H * W
    m_tiles = n * (hw // 128) if hw >= 128 else -(-n // (128 // hw))
    return (m_tiles + 1) // 2 * n_par * (cout // bn)


def min_many_tile_pairs(dev):
    """Fewest tile pairs that give every CTA at least three tiles, so that the second-and-later-tile paths of the
    persistent convolution (ring hand-over, staging toggles, next-tile prefetch) run twice.  The launcher uses at
    most multi_processor_count / 2 clusters; fewer resident clusters only add rounds.

    A CTA's later tiles are its first tile + k * clusters, so it only moves to another N-tile (and reloads the
    per-channel bias / GroupNorm / pose-bias parameters) when n_tiles does not divide the cluster count: with 66
    clusters, shapes of 1, 2, 3 or 6 N-tiles keep every CTA on one N-tile, 4, 5 or 8 do not."""
    return 3 * (torch.cuda.get_device_properties(dev).multi_processor_count // 2) + 1


def rounds(pairs, dev):
    """tiles each CTA runs (at most; fewer resident clusters only add rounds): ceil(pairs / clusters)"""
    clusters = torch.cuda.get_device_properties(dev).multi_processor_count // 2
    return -(-pairs // clusters)


def worst_block_rel_l2(out, ref, block=None):
    """-> (max rel-L2 over blocks, index of the worst block).  Blocks are the images of [n, C, ...] tensors, each
    split into `block`-channel slices when given (block = N-tile width: one block per (image, N-tile), the unit a
    wrong tile of the convolution spoils), so one bad tile among hundreds is not averaged away.  Computed in
    float64 on out's device; the index is (image, N-tile) with `block`, else the image."""
    out = out.detach().to(ref.device).double()
    ref = ref.detach().double()
    n, c = ref.shape[:2]
    nb = c // block if block else 1
    d = (out - ref).reshape(n, nb, -1).norm(dim=2)
    r = ref.reshape(n, nb, -1).norm(dim=2).clamp_min(1e-30)
    e = (d / r).flatten()
    i = int(e.argmax())
    return float(e[i]), ((i // nb, i % nb) if block else i)


def skip_without_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@contextlib.contextmanager
def no_host_sync():
    """torch raises on any host synchronisation inside the block (sync debug mode "error"); the device is synchronised
    first, and the mode is reset however the block ends"""
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(0)


def count_host_syncs(fn):
    """(result, the host synchronisations torch's sync debug mode reports during fn())"""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return out, sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def same_bits(a, b):
    """a and b (torch tensors on any device, or numpy arrays) have the same dtype, shape and bytes"""
    a, b = (np.ascontiguousarray(x.detach().cpu().numpy() if torch.is_tensor(x) else x) for x in (a, b))
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------ convolution cases
def _g(seed):
    return torch.Generator().manual_seed(seed)


CONV_CASES = [
    # n, C0, C1, Cout, S, mode
    (2, 192, 0, 192, 32, "3x3"), (3, 192, 192, 192, 32, "3x3"), (3, 384, 192, 384, 16, "3x3"),
    (5, 768, 384, 768, 8, "3x3"), (9, 1536, 768, 1536, 4, "3x3"), (2, 384, 0, 384, 16, "1x1"),
    (3, 128, 0, 192, 32, "1x1"), (3, 192, 192, 192, 32, "1x1"), (2, 192, 0, 192, 16, "unshuffle"),
    (5, 384, 0, 768, 4, "unshuffle"), (130, 768, 0, 12096, 1, "1x1"), (1, 64, 0, 64, 32, "3x3"),
    (3, 384, 0, 192, 32, "upsample3x3"), (5, 768, 0, 384, 16, "upsample3x3"),
    (7, 1536, 0, 768, 8, "upsample3x3"),
]


def conv_reference(x0, x1, w, b, mode):
    x = x0 if x1 is None else torch.cat([x0, x1], dim=1)
    if mode == "3x3":
        return F.conv2d(x, w, b, padding=1)
    if mode == "1x1":
        return F.conv2d(x, w, b)
    if mode == "upsample3x3":
        return F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, padding=1)
    n, c, hh, ww = x.shape
    x = x.reshape(n, c, hh // 2, 2, ww // 2, 2).permute(0, 1, 3, 5, 2, 4).reshape(n, c * 4, hh // 2, ww // 2)
    return F.conv2d(x, w, b)


def make_conv_case(n, C0, C1, Cout, S, mode, seed=0):
    g = _g(seed + n + C0 + Cout + S)
    cin = C0 + C1
    sin = 2 * S if mode == "unshuffle" else (S // 2 if mode == "upsample3x3" else S)
    x0 = h(torch.randn(n, C0, sin, sin, generator=g))
    x1 = h(torch.randn(n, C1, sin, sin, generator=g)) if C1 else None
    kk = {"3x3": 3, "1x1": 1, "unshuffle": 1, "upsample3x3": 3}[mode]
    cw = cin * 4 if mode == "unshuffle" else cin
    w = h(torch.randn(Cout, cw, kk, kk, generator=g) / (cw * kk * kk) ** 0.5)
    b = 0.1 * torch.randn(Cout, generator=g)
    return x0, x1, w, b


# ------------------------------------------------------------------ encoder inputs and module lists
def uniform_images(seed, B):
    g = torch.Generator().manual_seed(7000 + seed)
    return torch.rand((B, 3, 256, 256), generator=g) * 2 - 1


def crop_like_images(seed, B):
    """mostly -1 background with a textured object in the middle, as the model's crops are"""
    g = torch.Generator().manual_seed(8000 + seed)
    x = torch.full((B, 3, 256, 256), -1.0)
    yy, xx = torch.meshgrid(torch.arange(256.0), torch.arange(256.0), indexing="ij")
    for b in range(B):
        cy, cx, r = (torch.rand(3, generator=g) * torch.tensor([60.0, 60.0, 40.0]) + torch.tensor([98.0, 98.0, 50.0]))
        m = ((yy - cy) ** 2 + (xx - cx) ** 2) < r * r
        x[b][:, m] = torch.rand((3, int(m.sum())), generator=g) * 1.6 - 0.8
    return x


def mixed_images(n, seed):
    """n - n // 2 uniform images, then n // 2 crop-like ones"""
    return torch.cat([uniform_images(seed, n - n // 2), crop_like_images(seed, n // 2)])


# diffusers' AutoencoderKL config.json of Stable Diffusion v1.5's VAE
SD15_CONFIG = {
    "_class_name": "AutoencoderKL", "_diffusers_version": "0.6.0", "act_fn": "silu",
    "block_out_channels": [128, 256, 512, 512],
    "down_block_types": ["DownEncoderBlock2D", "DownEncoderBlock2D", "DownEncoderBlock2D", "DownEncoderBlock2D"],
    "in_channels": 3, "latent_channels": 4, "layers_per_block": 2, "norm_num_groups": 32, "out_channels": 3,
    "sample_size": 512,
    "up_block_types": ["UpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D"],
}

# the modules of the template encoder and the SD VAE encoder, in order, as the engines' run_block names them
ENC_MODULES = (["stem"] + [f"backbone.layer{l}.{b}" for l, n in ((1, 3), (2, 4), (3, 6), (4, 3)) for b in range(n)]
               + ["projector"])
VAE_MODULES = (["encoder.conv_in"]
               + [m for i in range(4) for m in [f"encoder.down_blocks.{i}.resnets.{j}" for j in range(2)]
                  + ([f"encoder.down_blocks.{i}.downsamplers.0"] if i < 3 else [])]
               + ["encoder.mid_block.resnets.0", "encoder.mid_block.attentions.0", "encoder.mid_block.resnets.1",
                  "encoder.conv_out"])


# ------------------------------------------------------------------ the split-precision engines one module at a time
# Worst per-image rel-L2 of one module against the float64 oracle.  Measured on an H100 80GB HBM3 at a 700 W power
# limit, over every module at n = 1, 3 and the chunk: template encoder worst 1.29e-5 (projector), median 4.9e-6; VAE
# encoder worst 1.70e-5 (down_blocks.2.downsamplers.0), median 8.6e-6; VAE decoder worst 1.71e-5
# (mid_block.resnets.0), median 8.1e-6.  The error follows K (fp32 tensor-core accumulation over up to 13 824
# products), above the ~1e-6 of the dropped A_lo W_lo term.  The gate is 2.6x the worst rather than 3x so that fp16
# inputs (2.0-2.9e-4 on test_split_precision_blocks_gpu's SENSITIVE modules) miss it by at least 4x.
SPLIT_BLOCK_TOL = 4.5e-5

ENC_CHUNK, VAE_CHUNK, DEC_CHUNK = 32, 16, 8


def run_block(engine, name, x):
    """-> (fp32 output, hi + lo of the pair or None)"""
    if isinstance(engine, torch.nn.Module):
        return engine.run_block(name, x), None
    return engine.run_block(name, x, want_pair=not name.endswith("conv_out"))


def encoder_weights(full):
    """the template encoder's weights of a full state_dict"""
    return {k[len("encoder."):]: v for k, v in full.items()
            if k.startswith("encoder.backbone.") or k.startswith("encoder.projector.")}


def encoder_taps(enc_sd):
    """the float64 oracle's (input, output) of every template encoder module on ENC_CHUNK seeded images"""
    skip_without_gpu()
    from oracle import unet_oracle
    taps = {}
    unet_oracle.encode_image({k: v.cuda().double() for k, v in enc_sd.items()},
                             mixed_images(ENC_CHUNK, 70).cuda().double(), taps=taps)
    return taps


def vae_encoder_taps(vae_sd):
    """the float64 oracle's (input, output) of every SD VAE encoder module on VAE_CHUNK seeded images"""
    skip_without_gpu()
    from oracle import vae_oracle
    taps = {}
    vae_oracle.encode(vae_sd, mixed_images(VAE_CHUNK, 71).cuda().double(), taps=taps)
    return taps
