"""GPU: the multi-GPU sweep (nope_b200.dist.ShardedSweep) on one GPU, W ranks simulated in one process.

torch.distributed is replaced by fakes for the calls nope_b200.dist makes: the rank and world size of the
simulated rank, and an all-gather that runs in two passes -- the first records every rank's packed record, the
second hands each rank the W recorded records back to back, as the collective would.  Every rank must then return
the sim and topi of one un-sharded sweep bit for bit (the CUDA merge kernel on real records), the ranks' local
template slices must make up the un-sharded templates, and each rank's record must come out the same in both
passes.  tools/dist_check.py is the same check on real GPUs under torchrun."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

pytestmark = pytest.mark.gpu


def _words(t):
    """the bit pattern of a float32 record (its int64 block reads as NaN floats)"""
    return t.view(torch.int32)


def sharded_sweeps(monkeypatch, engine, world, rf, poses, qf, **kw):
    """ShardedSweep.sweep on every rank of a simulated world, twice (record, then deliver) -> the per-rank outputs
    of the second pass"""
    from nope_b200.dist import ShardedSweep
    rank = {"r": 0}
    sent = [None] * world
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: rank["r"])
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)

    def record(recv, send, group=None):
        sent[rank["r"]] = send.clone()
        recv.zero_()

    def deliver(recv, send, group=None):
        assert torch.equal(_words(send), _words(sent[rank["r"]])), rank["r"]
        recv.copy_(torch.cat(sent))

    for fake in (record, deliver):
        monkeypatch.setattr(dist, "all_gather_into_tensor", fake)
        outs = []
        for r in range(world):
            rank["r"] = r
            outs.append(ShardedSweep().sweep(engine, rf, poses, qf, **kw))
    return outs


def check_ranks(outs, single, N, want_sim):
    embs = []
    for r, (sim, topi, (emb, lo, hi)) in enumerate(outs):
        assert torch.equal(topi, single["topi"]), r
        if want_sim:
            assert torch.equal(sim, single["sim"]), r
        else:
            assert sim is None
        if hi > lo:
            embs.append(emb)
        else:
            assert emb is None
        assert lo == (outs[r - 1][2][2] if r else 0), r                   # the slices tile the grid in order
    assert outs[-1][2][2] == N
    assert torch.equal(torch.cat(embs, dim=1), single["emb"])


def _poses(N, B):
    from nope_b200.poses import synthetic_pose_batch
    if N == 643:
        p, _ = synthetic_pose_batch(642, B)
        return torch.cat([p, p[:, :1]], dim=1)
    return synthetic_pose_batch(N, B)[0]


CASES = [(N, W, Q, want_sim, metric)
         for N, W in ((5, 8), (26, 3), (643, 8)) for Q in (1, 2) for want_sim in (True, False)
         for metric in ("l2", "cosine")]
CASES += [(10248, 8, 1, True, "l2"), (10248, 8, 2, False, "cosine")]


@pytest.mark.parametrize("N,W,Q,want_sim,metric", CASES)
def test_sharded_sweep_equals_single_sweep(gpu_model, monkeypatch, N, W, Q, want_sim, metric):
    """N = 5 on 8 ranks: one-pose and empty shards, k > shard size (the fill_record path); 643: a short last
    shard; 10 248 on 8 ranks: 1281-pose shards, the record length that once misaligned every second record."""
    u = gpu_model.u_net
    k = 5
    B = 1 if N == 10248 else 2
    g = torch.Generator().manual_seed(N + Q)
    rf = torch.randn(B, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn((B, Q, 8, 32, 32) if Q > 1 else (B, 8, 32, 32), generator=g) * 1.5
    poses = _poses(N, B)
    try:
        u.set_metric(metric)
        single = u.sweep(rf, poses, query_feat=qf, want_emb=True, k=k)
        outs = sharded_sweeps(monkeypatch, u, W, rf.cuda(), poses.cuda(), qf.cuda(), k=k, metric=metric,
                              want_emb=True, want_sim=want_sim)
    finally:
        u.set_metric("l2")
    check_ranks(outs, single, N, want_sim)


def test_sharded_ldm_sweep_equals_single_sweep(golden_dir, monkeypatch):
    """the LDM engine (UNetModelPose) through the same path: 7 poses on 4 ranks, two-pose shards and k = 5 > 2"""
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict
    m = UNetModelPose(device="cuda:0", chunk=2).load_state_dict(make_ldm_state_dict(seed=0))
    ref = torch.from_numpy(np.load(f"{golden_dir}/ldm_b1_n3.npz")["ref_latent"])
    g = torch.Generator().manual_seed(5)
    qry = torch.randn((1, 2) + tuple(ref.shape[1:]), generator=g)
    poses = _poses(7, 1)
    single = m.sweep(ref, poses, qry, want_emb=True, k=5)
    outs = sharded_sweeps(monkeypatch, m, 4, ref.cuda(), poses.cuda(), qry.cuda(), k=5, want_emb=True)
    check_ranks(outs, single, 7, True)
