"""GPU: every HBM-bound kernel of the UNet, one layer at a time,
through the C ABI, against the oracle's torch-fp32 restatement of the same reference op.
Inputs are pre-rounded to fp16 (the storage precision) so the comparison isolates the
kernel arithmetic; tolerances are stated per test."""
import pytest
import torch
import torch.nn.functional as F

from _util import h, log, rel_l2

pytestmark = pytest.mark.gpu

FP16_TOL = 1.5e-3     # rel-L2 of an fp16-stored result (one rounding = 4.9e-4 per element)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


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
