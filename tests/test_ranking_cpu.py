"""CPU: the ranking order every oracle states and every ranking kernel is held to (SURVEY.md section 7): descending
score; equal scores -- +0 and -0, inf and inf -- by the lowest index; NaN after every number, below -inf, and NaNs
among themselves by the lowest index; padding never ranked.  Small hand-written rows with the expected order written
out, so the oracles (and through tests/test_ranking_gpu.py the kernels) cannot drift from it."""
import torch

from oracle import hierarchy_oracle, inplane_refine_oracle, refine_oracle
from oracle import unet_oracle as orc

NAN, INF = float("nan"), float("inf")

# (row, its full order)
ROWS = [
    ([1.0, NAN, 3.0, -INF, 3.0], [2, 4, 0, 3, 1]),
    ([-0.0, 0.0, NAN, INF, NAN, INF, -1.0], [3, 5, 0, 1, 6, 2, 4]),
    ([0.0, -0.0, -INF, -INF, NAN], [0, 1, 2, 3, 4]),
    ([NAN, 2.0, NAN, 2.0, -2.0, 2.0], [1, 3, 5, 4, 0, 2]),
    ([NAN, NAN, NAN], [0, 1, 2]),
    ([-INF, -INF, -INF, -INF], [0, 1, 2, 3]),
]


def _same(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float32), torch.as_tensor(b, dtype=torch.float32)
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a[~a.isnan()], b[~b.isnan()]) and \
        torch.equal(torch.signbit(a[~a.isnan()]), torch.signbit(b[~b.isnan()]))


def test_topk_lowest_index():
    for row, order in ROWS:
        x = torch.tensor([row])
        for k in range(1, len(row) + 1):
            assert orc.topk_lowest_index(x, k)[0].tolist() == order[:k], (row, k)
        v, i = hierarchy_oracle.topk_lowest_index(x, len(row))
        assert i[0].tolist() == order and _same(v[0], [row[j] for j in order]), row


def test_cells_rank_orders_by_fine_index():
    """the candidates' fine indices, not their slots, break ties; padding (-1) is never ranked, however high its
    score; ranks past the candidates are (-inf, -1)"""
    sim = torch.tensor([[1.0, NAN, 3.0, 100.0, -INF, 3.0, NAN],
                        [NAN, NAN, 5.0, -0.0, 0.0, 7.0, 7.0]])
    cand = torch.tensor([[9, 2, 4, -1, 7, 0, 5],
                         [8, 3, 1, 6, 2, -1, -1]], dtype=torch.int32)
    full, v, i = hierarchy_oracle.rank(sim, cand, 10, 8)
    assert i.tolist() == [[0, 4, 9, 7, 2, 5, -1, -1], [1, 2, 6, 3, 8, -1, -1, -1]]
    assert _same(v[0], [3.0, 3.0, 1.0, -INF, NAN, NAN, -INF, -INF])
    assert _same(v[1], [5.0, 0.0, -0.0, NAN, NAN, -INF, -INF, -INF])
    assert _same(full[1], [-INF, 5.0, 0.0, NAN, -INF, -INF, -0.0, -INF, NAN, -INF])


def test_refine_select_with_infinite_threshold_is_the_order():
    """with trace_threshold = +inf nothing is suppressed: the select is the order over the non-padding slots"""
    for row, order in ROWS:
        n = len(row)
        sim = torch.tensor([row + [100.0]])                                  # a padding slot with the best score
        seed = torch.tensor([[10 + j for j in range(n)] + [-1]], dtype=torch.int32)
        cand = {"D": torch.randn(1, n + 1, 9), "rel": torch.randn(1, n + 1, 9), "seed": seed}
        out = refine_oracle.select(sim, cand, INF, n + 1)
        assert out["seed"][0].tolist() == [10 + j for j in order] + [-1], row
        assert _same(out["score"][0], [row[j] for j in order] + [-INF]), row


def test_inplane_select_with_infinite_threshold_is_the_order():
    """one centre: 3 angle slots x 9 pose slots, pair m = a * 9 + p"""
    flat = [-5.0] * 27
    for m, v in ((4, NAN), (20, 2.0), (7, 2.0), (0, -0.0), (26, 0.0), (13, INF), (1, NAN), (11, -INF)):
        flat[m] = v
    cand = {"D": torch.randn(1, 9, 9), "rel": torch.randn(1, 9, 9), "seed": torch.arange(10, 19).int()[None],
            "cossin": torch.tensor([[[1.0, 0.0], [0.6, 0.8], [0.6, -0.8]]])}
    out = inplane_refine_oracle.select(torch.tensor(flat).reshape(1, 3, 9), cand, INF, 27)
    m = (out["aslot"][0] * 9 + out["seed"][0] - 10).tolist()
    fives = [j for j in range(27) if flat[j] == -5.0]
    assert m == [13, 7, 20, 0, 26] + fives + [11, 1, 4]
    assert _same(out["score"][0], [flat[j] for j in m])


def test_merge_topk_order_and_padding():
    """the torch restatement of the multi-GPU merge: padding (-1) ranks after every candidate, NaN and -inf
    included (it is never a result while the ranks hold k valid candidates between them)"""
    from nope_b200.dist import merge_topk
    vals = torch.tensor([[1.0, -INF], [NAN, NAN], [3.0, 2.0], [-INF, NAN], [3.0, 2.0], [7.0, 9.0], [-0.0, 0.0]])
    idx = torch.tensor([[9, 5], [2, 3], [4, 8], [7, 1], [0, 6], [-1, -1], [11, 2]])
    v, i = merge_topk(vals, idx, 7)
    assert i.tolist() == [[0, 4, 9, 11, 7, 2, -1], [6, 8, 2, 5, 1, 3, -1]]
    assert _same(v[0], [3.0, 3.0, 1.0, -0.0, -INF, NAN, -INF])
    assert _same(v[1], [2.0, 2.0, 0.0, -INF, NAN, NAN, -INF])
    for row, order in ROWS:                                                  # one row split over two "ranks"
        h = (len(row) + 1) // 2
        vals = torch.tensor(row[:h] + [-INF] + row[h:] + [-INF])[:, None]
        idx = torch.tensor(list(range(h)) + [-1] + list(range(h, len(row))) + [-1])[:, None]
        v, i = merge_topk(vals, idx, len(row))
        assert i[0].tolist() == order, row
