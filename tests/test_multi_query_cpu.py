"""CPU: the multi-query surface (Q queries per reference sharing one sweep) without a device -- the batch
rules of the Python layer, argument validation in the library, and the sharded
merge with one record row per (reference, query) pair under gloo."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
def _fake():
    return C.c_void_p(256)       # never dereferenced: every call below fails its argument checks first


def _score_multi(B, Q, Bt, N, k):
    from nope_b200 import _lib
    lib = _lib.load()
    rc = lib.nope_score_topk_multi(_fake(), _fake(), B, Q, Bt, N, 8, 1024, 0, 0.2, k, _fake(), _fake(), _fake(),
                                   0, None)
    return rc, lib.nope_last_error().decode()


def test_score_topk_multi_rejects_bad_arguments():
    rc, msg = _score_multi(2, 0, 2, 26, 5)
    assert rc != 0 and "Q" in msg
    rc, msg = _score_multi(3, 1, 2, 26, 5)
    assert rc != 0 and "Bt" in msg
    rc, msg = _score_multi(1, 4, 1, 4, 5)
    assert rc != 0 and "k must be" in msg
    rc, msg = _score_multi(1, 4, 1, 100, 65)
    assert rc != 0 and "k must be" in msg


def test_sweep_multi_rejects_a_missing_engine():
    from nope_b200 import _lib
    lib = _lib.load()
    for fn in (lib.nope_unet_sweep_multi, lib.nope_ldm_sweep_multi):
        rc = fn(None, _fake(), _fake(), 1, 6, _fake(), 0, None, None, 0, None, None, 0, None)
        assert rc != 0 and len(lib.nope_last_error()) > 0


def test_broadcast_rule():
    """retrieval's [Bq] queries against [Bt, N] templates, as torch broadcasts the reference's
    query_feat.unsqueeze(1).repeat(1, N, ...) - template_feat (model.py:260-262)"""
    from nope_b200.model import broadcast_batches
    assert broadcast_batches(4, 4) == (4, 1, 4, 4)       # pairwise, as before
    assert broadcast_batches(16, 1) == (1, 16, 1, 16)    # one template set, many queries
    assert broadcast_batches(1, 3) == (3, 1, 3, 3)       # one query, several template sets
    assert broadcast_batches(1, 1) == (1, 1, 1, 1)
    for bq, bt in ((3, 2), (2, 3), (0, 1)):
        with pytest.raises(ValueError):
            broadcast_batches(bq, bt)
    # the restatement the rule follows: torch broadcasting of the difference tensor
    for bq, bt in ((4, 4), (16, 1), (1, 3)):
        d = torch.zeros(bq, 2, 3, 3)[:, None].expand(bq, 5, 2, 3, 3) - torch.zeros(bt, 5, 2, 3, 3)
        assert d.shape[0] == broadcast_batches(bq, bt)[3]


def test_score_topk_batch_mismatch_raises_before_touching_a_device():
    from nope_b200.model import score_topk
    with pytest.raises(ValueError, match="broadcast"):
        score_topk(torch.zeros(3, 8, 32, 32), torch.zeros(2, 26, 8, 32, 32))
    with pytest.raises(ValueError):
        score_topk(torch.zeros(2, 4, 32, 32), torch.zeros(2, 26, 8, 32, 32))


def test_query_forms():
    import types
    from nope_b200.ldm import UNetModelPose
    from nope_b200.model import PoseConditional
    from nope_b200.search import multi_query_form, query_rows
    ref = torch.zeros(2, 3, 8, 8)
    q, sq = multi_query_form(torch.zeros(2, 3, 8, 8), ref)          # one query per reference
    assert q.shape == (2, 3, 8, 8) and not sq
    q, sq = multi_query_form(torch.zeros(2, 5, 3, 8, 8), ref)       # Q = 5 per reference
    assert q.shape == (2, 5, 3, 8, 8) and not sq
    q, sq = multi_query_form(torch.zeros(7, 3, 8, 8), ref[:1])      # broadcast form: one reference
    assert q.shape == (1, 7, 3, 8, 8) and sq
    # the grid search of both front ends refuses these forms before any encoder call or sweep
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    ldm = UNetModelPose(device="cpu")
    rel, tp = torch.zeros(2, 6, 6), torch.zeros(6, 3, 3)
    for bad, r in ((torch.zeros(3, 3, 8, 8), ref), (torch.zeros(2, 0, 3, 8, 8), ref),
                   (torch.zeros(1, 5, 3, 8, 8), ref), (torch.zeros(2, 5, 4, 8, 8), ref)):
        for search in (multi_query_form, lambda q, r: model.predict_pose(q, r, rel, tp),
                       lambda q, r: ldm.predict_pose(q, r, rel, tp)):
            with pytest.raises(ValueError):
                search(bad, r)
    f = torch.zeros(2, 8, 32, 32)
    assert query_rows(torch.zeros(2, 8, 32, 32), f) == (1, (2,))
    assert query_rows(torch.zeros(2, 4, 8, 32, 32), f) == (4, (2, 4))
    for bad in (torch.zeros(2, 0, 8, 32, 32), torch.zeros(3, 8, 32, 32), torch.zeros(2, 4, 8, 16, 32)):
        with pytest.raises(ValueError):
            query_rows(bad, f)


def _worker(rank, world, port, B, Q, n_poses, k, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from nope_b200.dist import ShardedSweep, merge_topk, record_layout, shard_range
        from oracle.unet_oracle import topk_lowest_index
        g = torch.Generator().manual_seed(7)
        sim = torch.randn(B, Q, n_poses, generator=g)
        sim[0, 1, 4] = sim[0, 1, 2]                       # a tie across (possibly) different shards
        sim[B - 1, Q - 1, n_poses - 1] = sim[B - 1, Q - 1].max() + 1     # best in the last shard
        rows = B * Q
        flat = sim.reshape(rows, n_poses)
        lo, hi = shard_range(n_poses, rank, world)
        local = flat[:, lo:hi].contiguous()
        kl = min(k, hi - lo)
        if kl > 0:
            li = topk_lowest_index(local, kl)
            tv, ti = torch.gather(local, 1, li), li + lo
        else:
            tv, ti = torch.empty(rows, 0), torch.empty(rows, 0, dtype=torch.int64)
        ss = ShardedSweep()
        send, recv, topv_v, topi_v, off_s, pack, per = ss.record(rows, k, n_poses, True, torch.device("cpu"))
        assert (off_s, pack) == record_layout(rows, k, per, True)[1:]
        ss.fill_record(send, topv_v, topi_v, off_s, local, tv, ti)
        full, topi = ss.gather_merge(send, recv, rows, k, n_poses, per, pack, True)     # ONE all-gather
        ok = torch.equal(full.view(B, Q, n_poses), sim)
        ok = ok and torch.equal(topi.view(B, Q, k), topk_lowest_index(flat, k).view(B, Q, k))
        # merge_topk over the gathered candidates of every row gives the same ranking
        off_i = record_layout(rows, k, per, True)[0]
        rec = recv.view(world, pack)
        gv = rec[:, : rows * k].reshape(world, rows, k).permute(0, 2, 1).reshape(world * k, rows)
        gi = rec[:, off_i: off_i + 2 * rows * k].contiguous().view(torch.int64).view(world, rows, k) \
            .permute(0, 2, 1).reshape(world * k, rows)
        ok = ok and torch.equal(merge_topk(gv, gi, k)[1], topi)
        from nope_b200 import _lib
        ok = ok and pack == _lib.load().nope_topk_pack_floats(rows, k, per, 1)
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("B,Q,n_poses,k", [(2, 5, 26, 5), (1, 4, 642, 5), (3, 2, 7, 5)])
def test_multi_query_rows_gather_merge_gloo(B, Q, n_poses, k):
    world = 2
    port = 31500 + (os.getpid() + 7 * n_poses + Q) % 2000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, B, Q, n_poses, k, ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
