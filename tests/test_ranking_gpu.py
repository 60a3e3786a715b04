"""GPU: every ranking kernel against its oracle, bit for bit, on fp32 rows built on the host.

The order they all share (SURVEY.md section 7, DESIGN.md): descending score, equal scores (+0 == -0, inf == inf) by
the lowest index, NaN after every number and NaNs among themselves by index -- what a stable sort of -score gives.
Rows run from 1 to 92 232 entries (36 in-plane angles x 2562 poses), so the 256-thread loops hold several
candidates per thread; the value patterns aim at the per-thread running best, the warp butterfly and the cross-warp
pass of cta_argmax.  Indices are compared exactly, values bit for bit with NaN matched by position.  Also here: the
multi-GPU merge kernel on records laid out as ShardedSweep lays them out, and the score values of
nope_score_topk_multi at shapes the sweep never uses."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from _util import log
from oracle import hierarchy_oracle, inplane_refine_oracle, refine_oracle
from oracle import unet_oracle as orc

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
NS = (1, 5, 255, 256, 257, 642, 2562, 10248, 92232)
PATTERNS = ("random", "equal", "small_ints", "planted_ties", "signed_zero", "inf", "neg_inf_row",
            "nan_at_0", "nan_at_3", "nan_at_32", "nan_at_255", "nan_many", "nan_row")
IDX_BASES = (0, 2 ** 33 + 7)
ROWS = 3
SENTINEL = 1.0e30                  # never a value of any pattern: an output slot left unwritten shows up


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def make_rows(pattern, B, N, seed):
    """[B, N] float32 rows of one value pattern"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, generator=g)
    if pattern == "equal":                                   # pure index order
        x = torch.full((B, N), 0.75)
    elif pattern == "small_ints":                            # massive ties
        x = torch.randint(-2, 3, (B, N), generator=g).float()
    elif pattern == "planted_ties":
        # equal values at n and n + d: the same thread (d = 256), the same warp (1), different warps (32) and a
        # pair whose later index sits in a lower warp (224 wraps past the 256 threads); the pairs take the row's
        # best values, so every k sees them
        for b in range(B):
            top = float(x[b].max())
            for j, d in enumerate((256, 1, 32, 224)):
                if N > d:
                    n = int(torch.randint(0, N - d, (1,), generator=g))
                    x[b, n] = x[b, n + d] = top + 4 - j
    elif pattern == "signed_zero":
        x = -(x.abs() + 1)
        neg = torch.rand(B, N, generator=g) < 0.5
        zero = torch.rand(B, N, generator=g) < 0.125
        x = torch.where(zero, torch.where(neg, -0.0, 0.0), x)
        x[-1] = torch.where(neg[-1], -0.0, 0.0)              # a whole row of zeros of both signs
    elif pattern == "inf":
        pos = torch.randperm(N, generator=g)
        x[:, pos[: N // 3]] = -INF
        x[:, pos[N // 3: N // 3 + 2]] = INF
    elif pattern == "neg_inf_row":
        x = torch.full((B, N), -INF)
    elif pattern.startswith("nan_at_"):
        # one NaN at p, and the row's best values where a NaN that stuck as a thread's running best would hide
        # them: the same thread (p + 256, p + 512), the same warp (p + 1) and the next warp (p + 32)
        p = min(int(pattern[len("nan_at_"):]), N - 1)
        top = float(x.max())
        for j, q in enumerate((p + 256, p + 512, p + 1, p + 32)):
            if q < N:
                x[:, q] = top + 4 - j
        x[:, p] = NAN
    elif pattern == "nan_many":
        x[torch.rand(B, N, generator=g) < 0.1] = NAN
        x[0, 0] = NAN
    elif pattern == "nan_row":
        x = torch.full((B, N), NAN)
    else:
        assert pattern == "random", pattern
    return x.contiguous()


def ks(n, kmax=64):
    """k in {1, 5, 64} up to n, and k == n for short rows"""
    return sorted({k for k in (1, 5, 64) if k <= min(n, kmax)} | ({n} if n <= kmax else set()))


def same_bits(a, b):
    """bitwise equality of float32 tensors, NaNs matched by position (any payload)"""
    a, b = a.detach().cpu().float().contiguous(), b.detach().cpu().float().contiguous()
    if a.shape != b.shape:
        return False
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a.view(torch.int32)[~na], b.view(torch.int32)[~nb])


def oracle_topk(x, k):
    i = orc.topk_lowest_index(x, k)
    return x.gather(1, i), i


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _seed(*parts):
    """a generator seed per test case, the same in every process"""
    return zlib.crc32(repr(parts).encode())


# ------------------------------------------------------------------ nope_topk / the rank step of score_topk
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("N", NS)
def test_topk(dev, N, pattern):
    from nope_b200.model import topk
    x = make_rows(pattern, ROWS, N, _seed(N, pattern))
    for k in ks(N):
        ov, oi = oracle_topk(x, k)
        for base in IDX_BASES:
            v, i = topk(x.to(dev), k, idx_base=base)
            assert torch.equal(i.cpu(), oi + base), (k, base)
            assert same_bits(v, ov), (k, base)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("N", NS)
def test_score_topk_rank_step(dev, N, pattern):
    """The ranking of nope_score_topk_multi on the rows it scored: one channel, one pixel and the "l2" metric give
    sim = -(q - t)^2 per template, so the pattern's ties, infinities and NaNs reach the rank step; three query rows
    share one template batch (Bt = 1)."""
    from nope_b200.model import score_topk
    t = make_rows(pattern, 1, N, _seed(N, pattern)).reshape(1, N, 1, 1, 1)
    q = torch.tensor([0.0, 0.5, -1.0]).reshape(3, 1, 1, 1)
    for k in ks(N):
        for base in IDX_BASES:
            sim, i = score_topk(q.to(dev), t.to(dev), k=k, metric="l2", idx_base=base)
            sim = sim.cpu()
            assert torch.equal(sim.isnan(), t.reshape(1, N).isnan().expand(3, N)), (k, base)
            assert torch.equal(i.cpu(), orc.topk_lowest_index(sim, k) + base), (k, base)


# ------------------------------------------------------------------ coarse-to-fine rank
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("M", NS)
def test_cells_rank(dev, M, pattern):
    """nope_pose_cells_rank on candidate lists of distinct fine indices in any order: row 0 padded at its tail (as
    the expand kernel pads), row 1 with padding scattered through it, row 2 without padding.  k may exceed the
    number of candidates (the -inf / -1 ranks)."""
    from nope_b200.hierarchy import rank
    g = torch.Generator().manual_seed(_seed(M, pattern, "cells"))
    n_fine = M + M // 2 + 1
    sim = make_rows(pattern, ROWS, M, _seed(M, pattern))
    cand = torch.stack([torch.randperm(n_fine, generator=g)[:M] for _ in range(ROWS)]).to(torch.int32)
    cand[0, M - M // 5:] = -1
    cand[1, torch.randperm(M, generator=g)[: M // 3]] = -1
    for k in (1, 5, 64):
        full, v, i = rank(sim.to(dev), cand.to(dev), n_fine, k)
        full_o, v_o, i_o = hierarchy_oracle.rank(sim, cand, n_fine, k)
        assert torch.equal(i.cpu(), i_o), k
        assert same_bits(v, v_o), k
        assert same_bits(full, full_o), k


# ------------------------------------------------------------------ refinement selects
def _refine_cand(R, M, g):
    cand = {"D": torch.randn(R, M, 9, generator=g), "rel": torch.randn(R, M, 9, generator=g),
            "seed": torch.randint(0, 642, (R, M), generator=g, dtype=torch.int32)}
    cand["seed"][0, M - (M // 27) * 27 // 2:] = -1                          # padding centres at the tail
    cand["seed"][1, torch.randperm(M, generator=g)[: M // 5]] = -1          # padding anywhere
    return cand


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("M", (1, 5, 255, 256, 257, 642, 1728))
def test_refine_select(dev, M, pattern):
    """nope_pose_refine_select: with an infinite trace threshold it is a plain top-k over the non-padding slots;
    with a finite one (random rel matrices, traces ~ N(0, 9)) about a quarter of the candidates drop per pick."""
    from nope_b200.refine import select
    g = torch.Generator().manual_seed(_seed(M, pattern, "refine"))
    sim = make_rows(pattern, ROWS, M, _seed(M, pattern))
    cand = _refine_cand(ROWS, M, g)
    cand_d = {n: t.to(dev) for n, t in cand.items()}
    for thr in (INF, 2.0):
        for k in ks(M):
            out = select(sim.to(dev), cand_d, thr, k)
            out_o = refine_oracle.select(sim, cand, thr, k)
            for name in ("D", "seed", "rel"):
                assert torch.equal(out[name].cpu(), out_o[name]), (thr, k, name)
            assert same_bits(out["score"], out_o["score"]), (thr, k)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("keep", (1, 3, 4, 10, 16))
def test_inplane_select(dev, keep, pattern):
    """nope_pose_refine_inplane_select over keep * 3 angle slots x keep * 9 pose slots (27 to 6912 pairs per row):
    row 0 with scattered padding pose slots, row 1 with a padding centre (its pose slots and angle slots),
    row 2 entirely padding when keep == 1."""
    from nope_b200.inplane_refine import select
    g = torch.Generator().manual_seed(_seed(keep, pattern, "inplane"))
    P, A3 = keep * 9, keep * 3
    M = P * A3
    sim = make_rows(pattern, ROWS, M, _seed(M, pattern)).reshape(ROWS, A3, P)
    ang = torch.rand(ROWS, A3, generator=g) * 2 * math.pi
    cand = {"D": torch.randn(ROWS, P, 9, generator=g), "rel": torch.randn(ROWS, P, 9, generator=g),
            "seed": torch.randint(0, 642, (ROWS, P), generator=g, dtype=torch.int32),
            "cossin": torch.stack([ang.cos(), ang.sin()], dim=-1).float()}
    cand["seed"][0, torch.randperm(P, generator=g)[: P // 4]] = -1
    cand["seed"][1, (keep // 2) * 9: (keep // 2 + 1) * 9] = -1
    if keep == 1:
        cand["seed"][2] = -1
    cand_d = {n: t.to(dev) for n, t in cand.items()}
    for thr in (INF, 2.0):
        for k in ks(M):
            out = select(sim.to(dev), cand_d, thr, k)
            out_o = inplane_refine_oracle.select(sim, cand, thr, k)
            for name in ("D", "seed", "rel", "cossin", "aslot"):
                assert torch.equal(out[name].cpu(), out_o[name]), (thr, k, name)
            assert same_bits(out["score"], out_o["score"]), (thr, k)


# ------------------------------------------------------------------ multi-GPU merge
def _records(x, world, k, has_sim):
    """the W packed records of ShardedSweep.fill_record for rows x [B, N], back to back: each rank's oracle top
    min(k, n_local) with global indices, padded with (-inf, -1), then (has_sim) its slice of the rows.  Built as
    int32 words so every float and int64 bit pattern is copied exactly.  -> (gathered, per, pack)"""
    from nope_b200 import _lib
    from nope_b200.dist import record_layout, shard_range
    B, N = x.shape
    per = (N + world - 1) // world
    off_i, off_s, pack = record_layout(B, k, per, has_sim)
    assert pack == _lib.load().nope_topk_pack_floats(B, k, per, has_sim)
    rec = torch.zeros(world, pack, dtype=torch.int32)
    for r in range(world):
        lo, hi = shard_range(N, r, world)
        topv = torch.full((B, k), -INF)
        topi = torch.full((B, k), -1, dtype=torch.int64)
        kl = min(k, hi - lo)
        if kl > 0:
            v, i = oracle_topk(x[:, lo:hi], kl)
            topv[:, :kl], topi[:, :kl] = v, i + lo
        rec[r, : B * k] = topv.reshape(-1).view(torch.int32)
        rec[r, off_i: off_i + 2 * B * k] = topi.reshape(-1).view(torch.int32)
        if has_sim:
            rec[r, off_s: off_s + B * (hi - lo)] = x[:, lo:hi].contiguous().reshape(-1).view(torch.int32)
    return rec.reshape(-1).view(torch.float32), per, pack


@pytest.mark.parametrize("pattern", ("random", "equal", "small_ints", "signed_zero", "inf", "nan_at_3",
                                     "nan_many"))
@pytest.mark.parametrize("N", (5, 643, 10248))
@pytest.mark.parametrize("world", (1, 2, 3, 5, 8, 16))
def test_topk_merge(dev, world, N, pattern):
    """nope_topk_merge, driven directly: N = 5 leaves ranks empty, 643 makes the last rank short, 10 248 on 8 ranks
    is the 1281-pose shard that once misaligned every second record; B = 3 with odd k makes B * k odd (the pad
    float); world * k = 1024 is the shared-memory limit.  The outputs start as a sentinel, so a slot the kernel
    never writes fails."""
    from nope_b200 import _lib
    lib = _lib.load()
    for B in (1, 3):
        x = make_rows(pattern, B, N, _seed(N, pattern, B))
        for k in (1, 5, 64):
            if k > N or world * k > 1024:
                continue
            ov, oi = oracle_topk(x, k)
            for has_sim in (0, 1):
                gathered, per, pack = _records(x, world, k, has_sim)
                gathered = gathered.to(dev)
                out_sim = torch.full((B, N), SENTINEL, device=dev) if has_sim else None
                topv = torch.full((B, k), SENTINEL, device=dev)
                topi = torch.full((B, k), -7, device=dev, dtype=torch.int64)
                with torch.cuda.device(dev):
                    _lib.check(lib.nope_topk_merge(_lib.ptr(gathered), world, pack, B, k, N, per, has_sim,
                                                   _lib.ptr(out_sim), _lib.ptr(topv), _lib.ptr(topi), _stream(dev)))
                assert torch.equal(topi.cpu(), oi), (B, k, has_sim)
                assert same_bits(topv, ov), (B, k, has_sim)
                if has_sim:
                    assert same_bits(out_sim, x), (B, k)


# ------------------------------------------------------------------ score values
U = 2.0 ** -24                     # unit roundoff of fp32
SPATIAL = {1: (1, 1), 7: (1, 7), 300: (15, 20), 1024: (32, 32), 4096: (64, 64)}
BATCHES = ((1, 1), (2, 1), (5, 1), (2, 2), (1, 3))     # (query batch, template batch)
ORACLE = {"l2": orc.l2_similarity, "cosine": orc.cosine_similarity,
          "cosine_occlusion": orc.cosine_occlusion_similarity}


def rounding_depth(metric, Cc, hw):
    """the longest chain of fp32 roundings one term passes through in score_kernel: a thread's channel loop (Cc
    fused multiply-adds) and pixel loop (ceil(hw / 256) pixels), the warp butterfly (5) and the sum over the 8
    warps.  "cosine" runs one chain through all channels of all a thread's pixels; the other metrics finish each
    pixel's channel sum before they add the pixel."""
    px = math.ceil(hw / 256)
    return (Cc * px if metric == "cosine" else Cc + px) + 5 + 8


@pytest.mark.parametrize("Cc", (1, 3, 8, 16, 64))
@pytest.mark.parametrize("hw", tuple(SPATIAL))
@pytest.mark.parametrize("metric", tuple(ORACLE))
def test_score_values(dev, metric, hw, Cc):
    """nope_score_topk_multi's similarities against the oracle in float64 on the same fp32 inputs, for 1 to 5 query
    rows per template batch (the kernel's double-buffered partials cycle through them), a template batch of 1
    serving every query, and a query batch of 1 scored against several template batches.  Zero-norm pixels, a zero
    template and a zero query take the cosine metrics' eps branch."""
    from nope_b200.model import score_topk
    h, w = SPATIAL[hw]
    N, k = 7, 5
    d = rounding_depth(metric, Cc, hw)
    for Bq, Bt in BATCHES:
        g = torch.Generator().manual_seed(_seed(metric, hw, Cc, Bq, Bt))
        q = torch.randn(Bq, Cc, h, w, generator=g)
        t = torch.randn(Bt, N, Cc, h, w, generator=g) * 1.3 + 0.2
        t = t + torch.linspace(0, 3, N).view(1, N, 1, 1, 1) * q[:1, None]    # cosines from ~0 to near 1
        q[0, :, 0, 0] = 0.0                                   # a zero-norm query pixel
        t[..., -1, -1] = 0.0                                  # a zero-norm pixel in every template
        t[0, 1] = 0.0                                         # a whole zero template
        if Bq > 1:
            q[1] = 0.0                                        # a whole zero query
        sim, idx = score_topk(q.to(dev), t.to(dev), k=k, metric=metric)
        sim = sim.cpu().double()
        B = max(Bq, Bt)
        qd = q.double().expand(B, -1, -1, -1)
        td = t.double().expand(B, -1, -1, -1, -1)
        ref = ORACLE[metric](qd, td)
        if metric == "l2":
            # a sum of non-negative pixel terms: first-order bound d u |sum|, plus 8 u for the difference, the
            # squares and the square root of each pixel term
            bound = (d + 8) * U * ref.abs()
        else:
            # the dot product's error is d u sum|q t| <= d u |q| |t| by Cauchy-Schwarz, each norm adds d / 2 u, and
            # the square roots, the product and the division 4 u; per-pixel cosines in [-1, 1] and their mean
            # over hw stay within the same bound: an absolute error of (2 d + 8) u
            bound = torch.full_like(ref, (2 * d + 8) * U)
            if metric == "cosine_occlusion":
                # a pixel whose cosine lies within rounding of the 0.2 threshold may be kept by one side and
                # zeroed by the other: allow the threshold's worth for each such pixel
                pc = F.cosine_similarity(qd[:, None].expand_as(td), td, dim=2, eps=1e-8)
                near = ((pc - 0.2).abs() <= 4 * d * U).flatten(2).sum(dim=2)
                bound = bound + near * (0.2 + 4 * d * U) / hw
        err = (sim - ref).abs()
        log("score_values", metric=metric, hw=hw, C=Cc, Bq=Bq, Bt=Bt, max_err_over_bound=float((err / bound).max()))
        assert bool((err <= bound).all()), (Bq, Bt, float((err / bound).max()))
        assert torch.equal(idx.cpu(), orc.topk_lowest_index(sim.float(), k)), (Bq, Bt)
