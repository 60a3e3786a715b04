"""Multi-GPU sweep: the pose grid is embarrassingly parallel over hypotheses
(src/model/model.py:212-222 -- every (reference, pose) forward is independent), so rank g
takes a contiguous slice of the N poses with replicated weights and features, and the only
collective is ONE all-gather of a packed per-rank record -- local top-k scores, their GLOBAL
pose indices and (optionally) the rank's slice of the similarity row (SURVEY.md section 8e).
The sweep writes its outputs straight into the record, a single CUDA kernel (nope_topk_merge)
merges the gathered records, and the buffers are preallocated: no torch sort / gather / cat on
the path.  One process per GPU, torch.distributed (NCCL on GPUs; gloo in the CPU tests of the
collective plumbing, where the merge runs as the torch restatement `merge_topk`).  The reference
has no inference-time sharding; Lightning DDP there only shards the dataloader."""

import torch
import torch.distributed as dist

from . import _lib


def shard_range(n_poses, rank, world):
    """Contiguous slice [lo, hi) of rank `rank`; ceil(N/W) poses per rank, last may be short
    or empty."""
    per = (n_poses + world - 1) // world
    lo = min(rank * per, n_poses)
    return lo, min(lo + per, n_poses)


def record_layout(B, k, per, want_sim):
    """Offsets (in floats) of the packed record: topv | pad | topi (int64) | sim slice | pad, for B rows (a
    multi-query sweep has one row per (reference, query) pair: B = references * queries).
    The record length is a multiple of 4 floats: records sit back to back in the gathered buffer and the merge
    kernel reads the int64 indices of EVERY rank's record in place (an odd length -- e.g. the 10 248-pose grid on
    8 GPUs: 16 + 1281 floats -- put every second record's indices on a 4-byte boundary: misaligned address)."""
    kk = (B * k + 1) & ~1
    off_i, off_s = kk, kk + 2 * B * k
    return off_i, off_s, (off_s + (B * per if want_sim else 0) + 3) & ~3


def merge_topk(vals, idx, k):
    """Torch restatement of the merge rule (CPU tests; oracle of the CUDA kernel): vals/idx
    [W*k', B] candidates (any order, idx -1 = padding) -> top-k per batch row, descending score,
    ties -> lowest global index, NaN after every number; padding (-inf, -1) after every candidate."""
    vals = vals.clone()
    vals[idx < 0] = float("-inf")
    order = torch.sort(idx, dim=0, stable=True).indices           # ascending index first ...
    v1, i1 = torch.gather(vals, 0, order), torch.gather(idx, 0, order)
    order2 = torch.sort(-v1, dim=0, stable=True).indices          # ... then stable by score (NaN last) ...
    v2, i2 = torch.gather(v1, 0, order2), torch.gather(i1, 0, order2)
    order3 = torch.sort((i2 < 0).to(torch.uint8), dim=0, stable=True).indices     # ... then padding last
    v3, i3 = torch.gather(v2, 0, order3), torch.gather(i2, 0, order3)
    return v3[:k].t().contiguous(), i3[:k].t().contiguous()


class ShardedSweep:
    def __init__(self, group=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self._bufs = {}

    # ------------------------------------------------------------------ buffers
    def record(self, B, k, n_poses, want_sim, device):
        """Preallocated (send, recv) record buffers + views of the send record the sweep writes into."""
        per = (n_poses + self.world - 1) // self.world
        key = (B, k, per, bool(want_sim), str(device))
        if key not in self._bufs:
            off_i, off_s, pack = record_layout(B, k, per, want_sim)
            send = torch.zeros(pack, device=device, dtype=torch.float32)
            recv = torch.empty(self.world * pack, device=device, dtype=torch.float32)
            topv = send[: B * k].view(B, k)
            topi = send[off_i: off_i + 2 * B * k].view(torch.int64).view(B, k)
            self._bufs[key] = (send, recv, topv, topi, off_s, pack, per)
        return self._bufs[key]

    def gather_merge(self, send, recv, B, k, n_poses, per, pack, want_sim):
        """ONE all-gather of the packed records, then the merge.  -> (sim [B,N] | None, topi [B,k])."""
        dist.all_gather_into_tensor(recv, send, group=self.group)
        dev = send.device
        if dev.type == "cuda":
            sim = torch.empty((B, n_poses), device=dev, dtype=torch.float32) if want_sim else None
            topv = torch.empty((B, k), device=dev, dtype=torch.float32)
            topi = torch.empty((B, k), device=dev, dtype=torch.int64)
            with torch.cuda.device(dev):
                _lib.check(_lib.load().nope_topk_merge(
                    _lib.ptr(recv), self.world, pack, B, k, n_poses, per, 1 if want_sim else 0,
                    _lib.ptr(sim), _lib.ptr(topv), _lib.ptr(topi),
                    _lib.stream(dev)))
            return sim, topi
        # CPU (gloo) restatement: the collective plumbing tests
        off_i, off_s, _ = record_layout(B, k, per, want_sim)
        rec = recv.view(self.world, pack)
        gv = rec[:, : B * k].reshape(self.world, B, k).permute(0, 2, 1).reshape(self.world * k, B)
        gi = rec[:, off_i: off_i + 2 * B * k].contiguous().view(torch.int64).view(self.world, B, k) \
            .permute(0, 2, 1).reshape(self.world * k, B)
        _, topi = merge_topk(gv, gi, k)
        sim = None
        if want_sim:
            parts = []
            for r in range(self.world):
                lo, hi = shard_range(n_poses, r, self.world)
                parts.append(rec[r, off_s: off_s + B * (hi - lo)].view(B, hi - lo))
            sim = torch.cat(parts, dim=1).contiguous()
        return sim, topi

    def fill_record(self, send, topv_view, topi_view, off_s, local_sim, local_topv, local_topi):
        """Copy a rank's results into its record (used when the sweep could not write in place: k larger
        than the shard, or an empty shard); missing candidates are padding (-inf, -1)."""
        B, k = topv_view.shape
        topv_view.fill_(float("-inf"))
        topi_view.fill_(-1)
        if local_topv is not None and local_topv.numel() > 0:
            kl = local_topv.shape[1]
            topv_view[:, :kl] = local_topv
            topi_view[:, :kl] = local_topi
        if local_sim is not None and local_sim.numel() > 0:
            send[off_s: off_s + local_sim.numel()] = local_sim.reshape(-1)

    # ------------------------------------------------------------------ the sharded hot path
    def sweep(self, u_net, reference_feat, all_relativeR, query_feat, k=5, metric="l2",
              want_emb=False, want_sim=True, threshold=0.2):
        """-> (sim [B,N] | None, topi [B,k], emb).  `emb` (want_emb) is this rank's LOCAL slice
        [B, n_local, C, 32, 32] of the templates together with its pose range, as (emb, lo, hi):
        templates are never gathered (164 MB per query at N = 642).  query_feat [B,Q,C,32,32] (Q queries per
        reference) gives sim [B,Q,N] and topi [B,Q,k]: the B*Q (reference, query) pairs are the record's rows,
        still with one all-gather per sweep."""
        from .search import query_rows
        N = all_relativeR.shape[1]
        lo, hi = shard_range(N, self.rank, self.world)
        B = reference_feat.shape[0]
        Q, lead = query_rows(query_feat, reference_feat)
        rows = B * Q
        dev = u_net.device
        send, recv, topv_v, topi_v, off_s, pack, per = self.record(rows, k, N, want_sim, dev)
        emb = None
        n_local = hi - lo
        u_net.set_metric(metric, threshold)
        in_place = n_local >= k
        if in_place:
            poses = all_relativeR[:, lo:hi].contiguous()
            out = {"topv": topv_v.view(lead + (k,)), "topi": topi_v.view(lead + (k,))}
            if want_sim:
                out["sim"] = send[off_s: off_s + rows * n_local].view(lead + (n_local,))
            r = u_net.sweep(reference_feat, poses, query_feat=query_feat, want_emb=want_emb,
                            want_sim=want_sim, k=k, idx_base=lo, out=out)
            emb = r["emb"]
        elif n_local > 0:
            kl = min(k, n_local)
            poses = all_relativeR[:, lo:hi].contiguous()
            r = u_net.sweep(reference_feat, poses, query_feat=query_feat, want_emb=want_emb, k=kl, idx_base=lo)
            sim_l, tv, ti, emb = r["sim"], r["topv"].reshape(rows, kl), r["topi"].reshape(rows, kl), r["emb"]
            self.fill_record(send, topv_v, topi_v, off_s, sim_l if want_sim else None, tv, ti)
        else:
            self.fill_record(send, topv_v, topi_v, off_s, None, None, None)
        sim, topi = self.gather_merge(send, recv, rows, k, N, per, pack, want_sim)
        if len(lead) == 2:
            sim = sim.view(lead + (N,)) if sim is not None else None
            topi = topi.view(lead + (k,))
        return sim, topi, ((emb, lo, hi) if want_emb else None)
