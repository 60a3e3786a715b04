import json
import os

import torch

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
