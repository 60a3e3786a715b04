"""GPU: the clustered variant (conv_tc2.cuh, fused epilogues) of the wgmma convolution
against the same oracle and cases as the 1-CTA kernel, including odd tile counts (the
peer CTA of the last pair runs on a fully out-of-range tile) and fused GroupNorm statistics."""
import pytest
import torch
import torch.nn.functional as F

from _util import log, max_rel, rel_l2
from test_ops_gpu import CONV_CASES, conv_reference, make_conv_case
from test_conv_tc_gpu import EXTRA, TOL

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


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


@pytest.mark.parametrize("n,C0,Cout,S,G", [(3, 192, 192, 32, 8), (5, 768, 768, 8, 8),
                                           (11, 1536, 1536, 4, 8), (9, 128, 1536, 4, 1)])
def test_conv_2cta_fused_stats(dev, n, C0, Cout, S, G):
    from nope_b200 import ops
    mode = "3x3" if C0 != 128 else "1x1"
    x0, x1, w, b = make_conv_case(n, C0, 0, Cout, S, mode, seed=4)
    g = torch.Generator().manual_seed(S + Cout)
    gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
    beta = 0.2 * torch.randn(Cout, generator=g)
    ref = F.silu(F.group_norm(conv_reference(x0, None, w, b, mode), G, gamma, beta, eps=1e-5))
    out = ops.conv_gn(x0.to(dev), w.to(dev), b.to(dev), gamma.to(dev), beta.to(dev), G, silu=True,
                      mode=mode, impl="tcgen05_2cta")
    e = rel_l2(out, ref)
    log("conv_gn_2cta", n=n, Cout=Cout, S=S, G=G, rel_l2=e)
    assert e < 2e-3


def test_2cta_matches_1cta_bitwise(dev):
    """same operands, same fp32 accumulation order per output -> identical fp16 results"""
    from nope_b200 import ops
    x0, x1, w, b = make_conv_case(5, 384, 192, 384, 16, "3x3", seed=11)
    a = ops.conv(x0.to(dev), w.to(dev), b.to(dev), x1.to(dev), mode="3x3", impl="tcgen05")
    c = ops.conv(x0.to(dev), w.to(dev), b.to(dev), x1.to(dev), mode="3x3", impl="tcgen05_2cta")
    log("conv_2cta_vs_1cta", equal=bool(torch.equal(a, c)), rel_l2=rel_l2(c, a))
    assert rel_l2(c, a) < 1e-4
