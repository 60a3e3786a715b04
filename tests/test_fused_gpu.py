"""GPU: the sweep's fused layer -- convolution with GroupNorm + SiLU + pose bias + residual in its
epilogue (GnFuse, csrc/conv_tc.cuh; ResnetBlock.forward / Block.forward, model_utils.py:237-279;
PreNorm / to_out of LinearAttention, model_utils.py:230, 393-418) -- one layer at a time through the
C ABI against torch fp32.  Covers every tile geometry of the UNet: images spanning 8 / 2 M-tiles
(statistics exchanged between CTAs), 2 / 8 images per tile, groups spanning several N-tiles
(GroupNorm(1) at 384..1536 channels), odd image counts (phantom peer tiles), the hoisted-prefix
residual mapping, and the three precision modes.

The kernel is persistent (tile pairs cluster, cluster + clusters, ...).  The first CASES run one tile
per CTA; MANY_TILES run at least three per CTA (asserted from the shape: n = 53 / 41 / 197 / 401 at
sides 32 / 16 / 8 / 4), which reaches what only runs from a CTA's second tile on: the channel-parameter
cache, the double-buffered staging, the next tile's residual / pose-bias prefetch and several GroupNorm
sync groups per launch.  Errors are the worst rel-L2 over (image, N-tile) blocks, against float64."""
import pytest
import torch
import torch.nn.functional as F

from _util import h, log, max_rel, min_many_tile_pairs, pair_tiles, pick_bn, rounds, worst_block_rel_l2

pytestmark = pytest.mark.gpu

# one fp16 rounding of the stored output is 2.8e-4 rms; operands are pre-rounded in modes 0 / 1
TOL = {0: 6e-4, 1: 6e-4, 2: 3e-5}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


CASES = [
    # mode, n, C0, C1, Cout, S, G, silu, pb, res, res_div
    ("3x3", 5, 192, 0, 192, 32, 8, True, True, False, 0),     # block1 at 32^2: 8 tiles per image
    ("3x3", 5, 192, 0, 192, 32, 8, True, False, True, 0),     # block2 + identity residual
    ("3x3", 3, 192, 192, 192, 32, 8, True, True, False, 0),   # ups.3 concat input
    ("3x3", 6, 192, 0, 192, 32, 8, True, False, True, 3),     # downs.0.0: residual of the hoisted prefix
    ("3x3", 3, 384, 192, 384, 16, 8, True, True, True, 0),    # 2 tiles per image, 2 N-tiles
    ("3x3", 5, 768, 0, 768, 8, 8, True, True, True, 0),       # 2 images per tile, odd count
    ("3x3", 11, 768, 0, 1536, 4, 8, True, False, False, 0),   # 8 images per tile, ragged
    ("1x1", 3, 128, 0, 192, 32, 1, False, False, True, 0),    # to_out + GroupNorm(1) + residual
    ("1x1", 3, 128, 0, 384, 16, 1, False, False, True, 0),    # group spans 2 N-tiles x 2 M-tiles
    ("1x1", 5, 128, 0, 768, 8, 1, False, False, True, 0),     # group spans 4 N-tiles, 2 images per tile
    ("1x1", 9, 128, 0, 1536, 4, 1, False, False, True, 0),    # group spans 8 N-tiles, 8 images per tile
    ("1x1", 9, 128, 0, 1536, 4, 0, False, False, True, 0),    # mid_attn.to_out: residual only
    ("3x3", 2, 64, 0, 64, 32, 8, True, True, True, 0),        # u_net_dim 64: 64-wide tiles
    ("3x3", 3, 128, 0, 128, 16, 8, True, True, True, 0),      # u_net_dim 128: 128-wide tiles
    ("1x1", 3, 128, 0, 512, 4, 1, False, False, True, 0),     # 128-wide tiles, group over 4 N-tiles
    ("unshuffle", 3, 64, 0, 128, 16, 8, True, False, False, 0),
]
MANY_TILES = [
    # >= 3 tiles per CTA on 132 SMs (asserted from the shape).  Each pass-2 variant of the role-split epilogue
    # (conv_gn_math_warps) runs with and without emit, which selects a different variant: the first launch of
    # the test emits, the second does not and must reproduce it bit for bit.  Shapes with several N-tiles have
    # 4, 5 or 8 of them, counts that do not divide the 66 clusters: CTAs change N-tile between their tiles.
    ("3x3", 53, 64, 0, 192, 32, 8, True, True, False, 0),      # Block 1, table path: pose bias
    ("3x3", 53, 64, 0, 192, 32, 8, True, False, True, 0),      # Block 2, table path: residual
    ("3x3", 197, 128, 0, 768, 8, 8, True, True, False, 0),     # Block 1, 2 images per tile, phantom peer
    ("3x3", 197, 128, 0, 768, 8, 8, True, False, True, 0),     # Block 2, 2 images per tile, phantom peer
    ("3x3", 41, 64, 64, 640, 16, 10, True, True, True, 0),     # generic: two sources, pose bias + residual, 5 N-tiles
    ("3x3", 54, 64, 0, 192, 32, 8, True, False, True, 3),      # residual of the hoisted prefix
    ("1x1", 41, 128, 0, 640, 16, 1, False, False, True, 0),    # GroupNorm(1) over 5 N-tiles x 2 M-tiles
    ("1x1", 401, 128, 0, 1536, 4, 1, False, False, True, 0),   # GroupNorm(1) over 8 N-tiles, ragged
    ("3x3", 53, 64, 0, 128, 32, 8, True, True, True, 0),       # 128-wide tiles
    ("3x3", 53, 64, 0, 64, 32, 8, True, True, True, 0),        # 64-wide tiles
    ("unshuffle", 41, 64, 0, 640, 16, 10, True, False, False, 0),
    ("3x3", 11, 64, 0, 320, 32, 10, True, True, False, 0),     # 64-wide tiles over 5 N-tiles
]
CASES = CASES + MANY_TILES


def _reference(mode, x0, x1, w, b, gamma, beta, G, silu, cb, rs, res_div):
    x = x0 if x1 is None else torch.cat([x0, x1], 1)
    if mode == "unshuffle":
        bb, c, hh, ww = x.shape
        x = x.reshape(bb, c, hh // 2, 2, ww // 2, 2).permute(0, 1, 3, 5, 2, 4).reshape(bb, c * 4, hh // 2, ww // 2)
        y = F.conv2d(x, w, b)
    else:
        y = F.conv2d(x, w, b, padding=1 if mode == "3x3" else 0)
    if G > 0:
        y = F.group_norm(y, G, gamma, beta, eps=1e-5)
    if silu:
        y = F.silu(y)
    if cb is not None:
        y = y + cb[:, :, None, None]
    if rs is not None:
        idx = torch.arange(y.shape[0], device=y.device)
        idx = idx // res_div if res_div > 0 else idx
        y = y + rs[idx]
    return y


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(v) for v in c))
def test_conv_gn_fused(dev, case, precision):
    from nope_b200 import ops
    mode, n, C0, C1, Cout, S, G, silu, pb, res, res_div = case
    if precision == 1 and 3 < n and S == 32 and case not in MANY_TILES:
        pytest.skip("exact-weights mode covered by the smaller cases")
    pairs = pair_tiles(n, S, S, Cout, pick_bn(Cout))
    if case in MANY_TILES:
        assert pairs >= min_many_tile_pairs(dev), (case, pairs, "fewer than three tiles per CTA")
    g = torch.Generator().manual_seed(CASES.index(case) * 7 + 1)
    Sin = 2 * S if mode == "unshuffle" else S
    k = 3 if mode == "3x3" else 1
    cin_w = (C0 + C1) * (4 if mode == "unshuffle" else 1)
    r16 = (lambda t: t) if precision == 2 else h
    x0 = r16(torch.randn(n, C0, Sin, Sin, generator=g) * 1.2 + 0.2)
    x1 = r16(torch.randn(n, C1, Sin, Sin, generator=g)) if C1 else None
    w = torch.randn(Cout, cin_w, k, k, generator=g) / (cin_w * k * k) ** 0.5
    if precision == 0:
        w = h(w)
    b = 0.1 * torch.randn(Cout, generator=g)
    gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
    beta = 0.2 * torch.randn(Cout, generator=g)
    cb = h(torch.randn(n, Cout, generator=g)) if pb else None
    n_res = (n + res_div - 1) // res_div if res_div > 0 else n
    rs = r16(torch.randn(n_res, Cout, S, S, generator=g)) if res else None
    d64 = lambda t: None if t is None else t.to(dev, torch.float64)
    ref = _reference(mode, d64(x0), d64(x1), d64(w), d64(b), d64(gamma), d64(beta), G, silu, d64(cb), d64(rs), res_div)
    D = lambda t: None if t is None else t.to(dev)
    out, emit = ops.conv_gn_fused(D(x0), D(w), D(b), D(gamma), D(beta), groups=G, silu=silu, x1=D(x1), mode=mode,
                                  precision=precision, chan_bias=D(cb), residual=D(rs), res_div=res_div,
                                  want_emit=True)
    (e, blk), m = worst_block_rel_l2(out, ref, pick_bn(Cout)), max_rel(out, ref)
    # emitted GroupNorm(1) statistics = sums over the stored (fp16 hi) output
    o16 = out.cpu() if precision != 2 else out.cpu().half().float()
    es = torch.stack([o16.flatten(1).sum(1), (o16 ** 2).flatten(1).sum(1)], 1)
    e_emit = max_rel(emit, es)
    log("conv_gn_fused", case=list(case), precision=precision, pair_tiles=pairs, rounds=rounds(pairs, dev),
        n_tiles=Cout // pick_bn(Cout), worst_block_rel_l2=e,
        worst_block=blk, max_rel=m, emit_rel=e_emit)
    assert e < TOL[precision], (case, precision, "worst (image, N-tile)", blk, e)
    assert e_emit < 2e-3
    # bitwise reproducible, whatever the arrival order of the tiles
    out2 = ops.conv_gn_fused(D(x0), D(w), D(b), D(gamma), D(beta), groups=G, silu=silu, x1=D(x1), mode=mode,
                             precision=precision, chan_bias=D(cb), residual=D(rs), res_div=res_div)
    assert torch.equal(out2, out)


def test_fused_result_independent_of_batch_composition(dev):
    """An image's output must not depend on which other images share the launch (tile pairing,
    CTA assignment, arrival order): slices of a batch reproduce the full batch bit for bit."""
    from nope_b200 import ops
    g = torch.Generator().manual_seed(5)
    # n = 13: one tile per CTA; the larger n: >= 3 tiles per CTA, so slices start in the first, a middle and the
    # last round of the full launch
    for S, C, n, G in [(32, 192, 13, 8), (16, 384, 13, 8), (8, 768, 13, 8), (4, 1536, 13, 8),
                       (32, 192, 53, 8), (16, 640, 41, 10), (8, 768, 197, 8), (4, 1536, 401, 8)]:
        if n > 13:
            assert pair_tiles(n, S, S, C, pick_bn(C)) >= min_many_tile_pairs(dev), (S, C, n)
        x = h(torch.randn(n, C, S, S, generator=g))
        w = h(torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5)
        b = 0.1 * torch.randn(C, generator=g)
        gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
        cb = h(torch.randn(n, C, generator=g))
        D = lambda t: t.to(dev)
        run = lambda lo, hi: ops.conv_gn_fused(D(x[lo:hi]), D(w), D(b), D(gamma), D(beta), groups=G, silu=True,
                                               chan_bias=D(cb[lo:hi]), residual=D(x[lo:hi]))
        full = run(0, n)
        assert torch.equal(run(0, n), full), (S, C, n, "second launch")
        slices = [(0, 1), (3, 8), (12, 13), (5, 13)] if n == 13 else \
            [(0, 1), (n // 3, 2 * n // 3), (n - 1, n), ((n // 2) | 1, n)]
        for lo, hi in slices:
            part = run(lo, hi)
            if not torch.equal(part, full[lo:hi]):
                diff = (part != full[lo:hi]).flatten(1).any(1).nonzero().flatten() + lo
                raise AssertionError(f"S={S} C={C} n={n}: slice [{lo}, {hi}) differs from the full batch in "
                                     f"images {diff.tolist()[:8]}")
