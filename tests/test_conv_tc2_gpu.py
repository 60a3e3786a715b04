"""GPU: the clustered wgmma/TMA implicit-GEMM convolution (conv_tc2.cuh) against the oracle's torch-fp32
F.conv2d on the same fp16-rounded operands, for every geometry the UNet uses: 32/16/8/4 pixel sides (1, 1, 2
and 8 images per 128-row tile), two-source channel concatenation, 1x1, pixel-unshuffle + 1x1, the folded
nearest-x2 upsample, the 1x1-"image" linear layer, ragged last tiles, odd tile counts (the peer CTA of the
last pair runs on a fully out-of-range tile), all three N-tile widths, and the GroupNorm partial sums of the
plain epilogue."""
import pytest
import torch
import torch.nn.functional as F

from _util import log, max_rel, rel_l2
from test_ops_gpu import CONV_CASES, conv_reference, make_conv_case

pytestmark = pytest.mark.gpu

TOL = 1.5e-3   # rel-L2; fp32 accumulation, one fp16 rounding of the output


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


EXTRA = [(1, 128, 0, 128, 32, "3x3"), (4, 64, 64, 256, 8, "3x3"), (20, 1536, 0, 1536, 4, "3x3"),
         (300, 192, 0, 384, 4, "1x1")]


@pytest.mark.parametrize("n,C0,C1,Cout,S,mode", CONV_CASES + EXTRA)
def test_conv_2cta(dev, n, C0, C1, Cout, S, mode):
    from nope_b200 import ops
    x0, x1, w, b = make_conv_case(n, C0, C1, Cout, S, mode)
    ref = conv_reference(x0, x1, w, b, mode)
    out = ops.conv(x0.to(dev), w.to(dev), b.to(dev), None if x1 is None else x1.to(dev),
                   mode=mode, impl="tcgen05_2cta")
    e = rel_l2(out, ref)
    log("conv_2cta", n=n, C0=C0, C1=C1, Cout=Cout, S=S, mode=mode, rel_l2=e, max_rel=max_rel(out, ref))
    assert e < TOL


def test_conv_2cta_no_bias(dev):
    from nope_b200 import ops
    x0, x1, w, _ = make_conv_case(3, 192, 192, 384, 16, "3x3", seed=9)
    ref = conv_reference(x0, x1, w, None, "3x3")
    out = ops.conv(x0.to(dev), w.to(dev), None, x1.to(dev), mode="3x3", impl="tcgen05_2cta")
    e = rel_l2(out, ref)
    log("conv_2cta_no_bias", rel_l2=e, max_rel=max_rel(out, ref))
    assert e < TOL


@pytest.mark.parametrize("n,C0,C1,Cout,S,mode,G", [
    (3, 192, 0, 192, 32, "3x3", 8), (2, 384, 192, 384, 16, "3x3", 8), (5, 768, 0, 768, 8, "3x3", 8),
    (11, 1536, 0, 1536, 4, "3x3", 8), (3, 128, 0, 192, 32, "1x1", 1), (9, 128, 0, 1536, 4, "1x1", 1),
    (2, 64, 0, 64, 32, "3x3", 8)])
def test_conv_gn(dev, n, C0, C1, Cout, S, mode, G):
    """Block.forward: conv -> GroupNorm -> SiLU, normalised from nothing but the partial sums of the plain
    epilogue (32-row x 8-channel partials, every images-per-tile case incl. 2 images per warp at 4x4)."""
    from nope_b200 import ops
    x0, x1, w, b = make_conv_case(n, C0, C1, Cout, S, mode, seed=3)
    g = torch.Generator().manual_seed(S + Cout)
    gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
    beta = 0.2 * torch.randn(Cout, generator=g)
    ref = F.silu(F.group_norm(conv_reference(x0, x1, w, b, mode), G, gamma, beta, eps=1e-5))
    out = ops.conv_gn(x0.to(dev), w.to(dev), b.to(dev), gamma.to(dev), beta.to(dev), G, silu=True,
                      x1=None if x1 is None else x1.to(dev), mode=mode, impl="tcgen05_2cta")
    e = rel_l2(out, ref)
    log("conv_gn", n=n, Cout=Cout, S=S, G=G, rel_l2=e)
    assert e < 2e-3
