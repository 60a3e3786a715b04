"""GPU: the clustered wgmma/TMA implicit-GEMM convolution (conv_tc2.cuh) against F.conv2d in float64 on the same
fp16-rounded operands, for every geometry the UNet uses: 32/16/8/4 pixel sides (1, 1, 2 and 8 images per 128-row
tile), two-source channel concatenation, 1x1, pixel-unshuffle + 1x1, the folded nearest-x2 upsample, the 1x1-"image"
linear layer, ragged last tiles, odd tile counts (the peer CTA of the last pair runs on a fully out-of-range tile), all
three N-tile widths, and the GroupNorm partial sums of the plain epilogue.

The kernel is persistent: each 2-CTA cluster walks tile pairs cluster, cluster + clusters, ...  MANY_TILES cases
have enough tile pairs (asserted from the shape) that every CTA runs at least three tiles, so the paths that only
run from a CTA's second tile on -- ring phases, the epilogue-to-mainloop hand-over, the output staging toggle, the
next tile's prefetches -- are compared with the reference too.  Errors are the worst rel-L2 over (image, N-tile)
blocks, so one wrong tile among hundreds fails the test and is named."""
import pytest
import torch
import torch.nn.functional as F

from _util import (CONV_CASES, conv_reference, log, make_conv_case, max_rel, min_many_tile_pairs, pair_tiles, pick_bn,
                   rounds, worst_block_rel_l2)

pytestmark = pytest.mark.gpu

TOL = 1.5e-3   # rel-L2; fp32 accumulation, one fp16 rounding of the output


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def conv_pairs(n, Cout, S, mode):
    """tile pairs of the launch (output side S; the folded upsample tiles its source pixels, 4 parities)"""
    if mode == "upsample3x3":
        return pair_tiles(n, S // 2, S // 2, Cout, pick_bn(Cout), n_par=4)
    return pair_tiles(n, S, S, Cout, pick_bn(Cout))


def check_rounds(dev, case, pairs):
    assert pairs >= min_many_tile_pairs(dev), (case, pairs, "fewer than three tiles per CTA")


def _d64(dev, *ts):
    return [None if t is None else t.to(dev, torch.float64) for t in ts]


EXTRA = [(1, 128, 0, 128, 32, "3x3"), (4, 64, 64, 256, 8, "3x3"), (20, 1536, 0, 1536, 4, "3x3"),
         (300, 192, 0, 384, 4, "1x1")]
# >= 3 tiles per CTA on 132 SMs; few input channels keep the float64 reference cheap.  Where a shape has several
# N-tiles their count does not divide the 66 clusters (640 channels: 5 of 128), so CTAs change N-tile between tiles.
MANY_TILES = [
    (53, 64, 0, 192, 32, "3x3"), (41, 64, 64, 640, 16, "3x3"),
    (197, 128, 0, 768, 8, "3x3"),        # odd m-tile count: the peer of the last pair runs a phantom tile
    (401, 128, 0, 1536, 4, "3x3"),       # ragged last tile and a phantom peer
    (900, 128, 0, 12096, 1, "1x1"), (53, 128, 0, 192, 32, "1x1"), (41, 64, 0, 640, 16, "unshuffle"),
    (50, 64, 0, 192, 32, "upsample3x3"), (97, 128, 0, 384, 16, "upsample3x3"),
    (53, 64, 0, 128, 32, "3x3"), (53, 64, 0, 64, 32, "3x3"),
]


@pytest.mark.parametrize("n,C0,C1,Cout,S,mode", CONV_CASES + EXTRA + MANY_TILES)
def test_conv_2cta(dev, n, C0, C1, Cout, S, mode):
    from nope_b200 import ops
    case = (n, C0, C1, Cout, S, mode)
    pairs = conv_pairs(n, Cout, S, mode)
    if case in MANY_TILES:
        check_rounds(dev, case, pairs)
    x0, x1, w, b = make_conv_case(n, C0, C1, Cout, S, mode)
    ref = conv_reference(*_d64(dev, x0, x1, w, b), mode)
    out = ops.conv(x0.to(dev), w.to(dev), b.to(dev), None if x1 is None else x1.to(dev), mode=mode)
    e, blk = worst_block_rel_l2(out, ref, pick_bn(Cout))
    log("conv_2cta", n=n, C0=C0, C1=C1, Cout=Cout, S=S, mode=mode, pair_tiles=pairs, rounds=rounds(pairs, dev),
        n_tiles=Cout // pick_bn(Cout), worst_block_rel_l2=e,
        worst_block=blk, max_rel=max_rel(out, ref))
    assert e < TOL, (case, "worst (image, N-tile)", blk, e)


def _no_bias_case(dev, n, C0, C1, Cout=384):
    from nope_b200 import ops
    x0, x1, w, _ = make_conv_case(n, C0, C1, Cout, 16, "3x3", seed=9)
    ref = conv_reference(*_d64(dev, x0, x1, w), None, "3x3")
    out = ops.conv(x0.to(dev), w.to(dev), None, x1.to(dev), mode="3x3")
    e, blk = worst_block_rel_l2(out, ref, pick_bn(Cout))
    pairs = conv_pairs(n, Cout, 16, "3x3")
    log("conv_2cta_no_bias", n=n, Cout=Cout, pair_tiles=pairs, rounds=rounds(pairs, dev), worst_block_rel_l2=e,
        worst_block=blk, max_rel=max_rel(out, ref))
    assert e < TOL, (n, "worst (image, N-tile)", blk, e)
    return pairs


def test_conv_2cta_no_bias(dev):
    _no_bias_case(dev, 3, 192, 192)


def test_conv_2cta_no_bias_many_tiles(dev):
    """two sources and no bias with >= 3 tiles per CTA, 5 N-tiles"""
    check_rounds(dev, "no_bias", conv_pairs(41, 640, 16, "3x3"))
    _no_bias_case(dev, 41, 64, 64, 640)


GN_MANY_TILES = [(53, 64, 0, 192, 32, "3x3", 8), (197, 128, 0, 768, 8, "3x3", 8), (401, 128, 0, 1536, 4, "1x1", 1)]


@pytest.mark.parametrize("n,C0,C1,Cout,S,mode,G", [
    (3, 192, 0, 192, 32, "3x3", 8), (2, 384, 192, 384, 16, "3x3", 8), (5, 768, 0, 768, 8, "3x3", 8),
    (11, 1536, 0, 1536, 4, "3x3", 8), (3, 128, 0, 192, 32, "1x1", 1), (9, 128, 0, 1536, 4, "1x1", 1),
    (2, 64, 0, 64, 32, "3x3", 8)] + GN_MANY_TILES)
def test_conv_gn(dev, n, C0, C1, Cout, S, mode, G):
    """Block.forward: conv -> GroupNorm -> SiLU, normalised from nothing but the partial sums of the plain
    epilogue (32-row x 8-channel partials, every images-per-tile case incl. 2 images per warp at 4x4)."""
    from nope_b200 import ops
    case = (n, C0, C1, Cout, S, mode, G)
    pairs = conv_pairs(n, Cout, S, mode)
    if case in GN_MANY_TILES:
        check_rounds(dev, case, pairs)
    x0, x1, w, b = make_conv_case(n, C0, C1, Cout, S, mode, seed=3)
    g = torch.Generator().manual_seed(S + Cout)
    gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
    beta = 0.2 * torch.randn(Cout, generator=g)
    x0d, x1d, wd, bd, gd, btd = _d64(dev, x0, x1, w, b, gamma, beta)
    ref = F.silu(F.group_norm(conv_reference(x0d, x1d, wd, bd, mode), G, gd, btd, eps=1e-5))
    out = ops.conv_gn(x0.to(dev), w.to(dev), b.to(dev), gamma.to(dev), beta.to(dev), G, silu=True,
                      x1=None if x1 is None else x1.to(dev), mode=mode)
    e, blk = worst_block_rel_l2(out, ref, pick_bn(Cout))
    log("conv_gn", n=n, Cout=Cout, S=S, G=G, pair_tiles=pairs, rounds=rounds(pairs, dev), worst_block_rel_l2=e,
        worst_block=blk)
    assert e < 2e-3, (case, "worst (image, N-tile)", blk, e)
