"""GPU: every HBM-bound kernel and the SIMT twin of the convolution, one layer at a time,
through the C ABI, against the oracle's torch-fp32 restatement of the same reference op.
Inputs are pre-rounded to fp16 (the storage precision) so the comparison isolates the
kernel arithmetic; tolerances are stated per test."""
import pytest
import torch
import torch.nn.functional as F

from _util import h, log, max_rel, rel_l2

pytestmark = pytest.mark.gpu

FP16_TOL = 1.5e-3     # rel-L2 of an fp16-stored result (one rounding = 4.9e-4 per element)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("n,C,S,G,silu,bias,res", [
    (3, 192, 32, 8, True, True, True), (2, 384, 16, 8, True, False, False),
    (5, 768, 8, 8, True, True, False), (9, 1536, 4, 8, True, False, True),
    (2, 192, 32, 1, False, False, True), (3, 1536, 4, 1, False, False, False),
    (1, 64, 32, 8, True, True, True)])
def test_groupnorm(dev, n, C, S, G, silu, bias, res):
    from nope_b200 import ops
    g = _g(n * C + S)
    x = h(torch.randn(n, C, S, S, generator=g) * 1.3 + 0.4)
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    beta = 0.2 * torch.randn(C, generator=g)
    cb = h(torch.randn(n, C, generator=g)) if bias else None
    rs = h(torch.randn(n, C, S, S, generator=g)) if res else None
    ref = F.group_norm(x, G, gamma, beta, eps=1e-5)
    if silu:
        ref = F.silu(ref)
    if bias:
        ref = ref + cb[:, :, None, None]
    if res:
        ref = ref + rs
    out = ops.groupnorm(x.to(dev), gamma.to(dev), beta.to(dev), G, silu=silu,
                        chan_bias=None if cb is None else cb.to(dev),
                        residual=None if rs is None else rs.to(dev))
    e = rel_l2(out, ref)
    log("groupnorm", n=n, C=C, S=S, G=G, rel_l2=e)
    assert e < FP16_TOL


@pytest.mark.parametrize("n,S", [(3, 32), (2, 16), (5, 8), (7, 4)])
def test_linear_attention(dev, n, S):
    from nope_b200 import ops
    g = _g(S)
    qkv = h(torch.randn(n, 384, S, S, generator=g) * 1.5)
    b, hw = n, S * S
    q, k, v = [t.reshape(b, 4, 32, hw) for t in qkv.chunk(3, dim=1)]
    q = q.softmax(dim=-2) * 32 ** -0.5
    k = k.softmax(dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", k, v)
    ref = torch.einsum("bhde,bhdn->bhen", ctx, q).reshape(b, 128, S, S)
    out = ops.linear_attention(qkv.to(dev))
    e = rel_l2(out, ref)
    log("linear_attention", n=n, S=S, rel_l2=e)
    assert e < FP16_TOL


@pytest.mark.parametrize("n,S", [(3, 32), (5, 16), (150, 16), (1, 32)])
def test_linear_attention_tcgen05(dev, n, S):
    """The tensor-core LinearAttention core (csrc/linattn_tc.cuh): ek^T v and qs ctx as wgmma GEMMs over
    token-major operands (MN-major descriptors), exp / softmax transforms in place.  fp16 operands (ek, qs,
    ctx) add ~3e-4 to the one output rounding of the CUDA-core kernel."""
    from nope_b200 import ops
    g = _g(S + n)
    qkv = h(torch.randn(n, 384, S, S, generator=g) * 1.5)
    b, hw = n, S * S
    q, k, v = [t.reshape(b, 4, 32, hw).double() for t in qkv.chunk(3, dim=1)]
    q = q.softmax(dim=-2) * 32 ** -0.5
    k = k.softmax(dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", k, v)
    ref = torch.einsum("bhde,bhdn->bhen", ctx, q).reshape(b, 128, S, S)
    out = ops.linear_attention(qkv.to(dev), impl="tcgen05")
    e = rel_l2(out, ref)
    simt = ops.linear_attention(qkv.to(dev), impl="simt")
    log("linear_attention_tc", n=n, S=S, rel_l2=e, rel_l2_simt=rel_l2(simt, ref), vs_simt=rel_l2(out, simt))
    assert e < FP16_TOL
    assert torch.equal(ops.linear_attention(qkv.to(dev), impl="tcgen05"), out)     # deterministic


@pytest.mark.parametrize("n,S", [(6, 4), (2, 2)])
def test_attention(dev, n, S):
    from nope_b200 import ops
    g = _g(10 + S)
    qkv = h(torch.randn(n, 384, S, S, generator=g) * 1.5)
    hw = S * S
    q, k, v = [t.reshape(n, 4, 32, hw) for t in qkv.chunk(3, dim=1)]
    sim = torch.einsum("bhdi,bhdj->bhij", q * 32 ** -0.5, k)
    attn = (sim - sim.amax(dim=-1, keepdim=True)).softmax(dim=-1)
    ref = torch.einsum("bhij,bhdj->bhid", attn, v).permute(0, 1, 3, 2).reshape(n, 128, S, S)
    out = ops.attention(qkv.to(dev))
    e = rel_l2(out, ref)
    log("attention", n=n, S=S, rel_l2=e)
    assert e < FP16_TOL


def test_upsample(dev):
    from nope_b200 import ops
    x = h(torch.randn(3, 64, 8, 8, generator=_g(1)))
    out = ops.upsample2x(x.to(dev))
    assert torch.equal(out.cpu(), F.interpolate(x, scale_factor=2, mode="nearest"))


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


@pytest.mark.parametrize("n,C0,C1,Cout,S,mode", CONV_CASES)
def test_conv_simt(dev, n, C0, C1, Cout, S, mode):
    from nope_b200 import ops
    x0, x1, w, b = make_conv_case(n, C0, C1, Cout, S, mode)
    ref = conv_reference(x0, x1, w, b, mode)
    out = ops.conv(x0.to(dev), w.to(dev), b.to(dev), None if x1 is None else x1.to(dev),
                   mode=mode, impl="simt")
    e = rel_l2(out, ref)
    log("conv_simt", n=n, C0=C0, C1=C1, Cout=Cout, S=S, mode=mode, rel_l2=e, max_rel=max_rel(out, ref))
    assert e < FP16_TOL


@pytest.mark.parametrize("metric", ["l2", "cosine", "cosine_occlusion"])
def test_score_topk(dev, metric):
    from nope_b200.model import score_topk
    from oracle import unet_oracle as orc
    g = _g(5)
    q = torch.randn(3, 8, 32, 32, generator=g)
    t = torch.randn(3, 41, 8, 32, 32, generator=g)
    t[1, 7] = t[1, 3]                                  # exact tie -> lowest index wins
    ref = {"l2": orc.l2_similarity, "cosine": orc.cosine_similarity,
           "cosine_occlusion": orc.cosine_occlusion_similarity}[metric](q, t)
    sim, idx = score_topk(q.to(dev), t.to(dev), k=5, metric=metric)
    e = rel_l2(sim, ref)
    log("score_topk", metric=metric, rel_l2=e)
    assert e < 1e-5                                    # fp32 arithmetic, summation order only
    assert torch.equal(idx.cpu(), orc.topk_lowest_index(sim.cpu(), 5))
    assert sim[1, 7] == sim[1, 3]
    with pytest.raises(RuntimeError):
        score_topk(q.to(dev), t[:, :4].to(dev), k=5, metric=metric)   # torch.topk raises for N<5
    with pytest.raises(ValueError):
        score_topk(q.to(dev), t.to(dev), k=5, metric="dot")
