"""GPU: Q queries per reference sharing one sweep (nope_unet_sweep_multi / nope_ldm_sweep_multi /
nope_score_topk_multi and the Python forms above them).

Pinned here: a Q-query call is bit-identical to Q one-query calls (each (hypothesis, query) score is summed
in an order that does not depend on Q), a [B, 1, ...] query through the Python layer is bit-identical to a
[B, C, 32, 32] query through the C ABI, and the scores meet the same tolerances against the CPU oracle as the
single-query path (tests/test_unet_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from _util import log, max_rel

pytestmark = pytest.mark.gpu

SIM_TOL = 1e-3          # scores against the oracle, fp16 mode and parity mode (tests/test_unet_gpu.py)
METRICS = ("l2", "cosine", "cosine_occlusion")


def multi_queries(g, Q=5):
    """[B, Q, 8, 32, 32] queries per reference of the grid26_b2 fixture: the fixture's own query, blends of it
    with the reference and a seeded perturbation.  Chosen so that the oracle's adjacent top-6 scores are at
    least 3.4e-3 apart (relative), well above the fp16 mode's score error: the whole top-5 is pinned."""
    qf, rf = torch.from_numpy(g["query_feat"]), torch.from_numpy(g["ref_feat"])
    gen = torch.Generator().manual_seed(11)
    noise = torch.randn(qf.shape, generator=gen) * qf.std()
    cand = [qf, 0.75 * qf + 0.25 * rf, qf - 0.1 * noise, 0.25 * qf + 0.75 * rf, 0.5 * (qf + rf)]
    return torch.stack(cand[:Q], dim=1).contiguous()


def _direct_sweep(u, rf, poses, qf, k):
    """nope_unet_sweep_multi with Q = 1 and a [B, C, 32, 32] query, called directly through the C ABI"""
    from nope_b200 import _lib
    lib = _lib.load()
    dev = u.device
    rf, poses, qf = (t.to(dev, torch.float32).contiguous() for t in (rf, poses, qf))
    B, N = poses.shape[:2]
    sim = torch.empty((B, N), device=dev)
    topv = torch.empty((B, k), device=dev)
    topi = torch.empty((B, k), device=dev, dtype=torch.int64)
    u.reserve(min(u._chunk, B * N), B, B * N)
    with torch.cuda.device(dev):
        _lib.check(lib.nope_unet_sweep_multi(u._handle(), _lib.ptr(rf), _lib.ptr(poses), B, N, _lib.ptr(qf), 1,
                                             None, _lib.ptr(sim), k, _lib.ptr(topv), _lib.ptr(topi), 0,
                                             C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return sim, topv, topi


@pytest.mark.parametrize("metric", METRICS)
def test_q1_equals_single_query_entry_point(gpu_model, golden_dir, metric):
    g = np.load(f"{golden_dir}/level2_642_b1.npz")
    rf, qf = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["query_feat"])
    poses = torch.from_numpy(g["all_relativeR"])
    u = gpu_model.u_net
    try:
        u.set_metric(metric, 0.2)
        one = _direct_sweep(u, rf, poses, qf, 5)
        multi = u.sweep(rf, poses, query_feat=qf[:, None], want_emb=False, k=5)
    finally:
        u.set_metric("l2")
    assert multi["sim"].shape == (1, 1, 642) and multi["topi"].shape == (1, 1, 5)
    assert torch.equal(multi["sim"][:, 0], one[0])
    assert torch.equal(multi["topv"][:, 0], one[1])
    assert torch.equal(multi["topi"][:, 0], one[2])


@pytest.mark.parametrize("metric", METRICS)
def test_query_count_invariance(gpu_model, golden_dir, metric):
    """B = 2, N = 26, Q = 5: every sim[b, q] / topi[b, q] equals a one-query sweep of query q, bit for bit"""
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    rf, poses = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"])
    qs = multi_queries(g)
    u = gpu_model.u_net
    try:
        u.set_metric(metric, 0.2)
        out = u.sweep(rf, poses, query_feat=qs, want_emb=False, k=5)
        assert out["sim"].shape == (2, 5, 26) and out["topi"].shape == (2, 5, 5)
        for q in range(qs.shape[1]):
            one = u.sweep(rf, poses, query_feat=qs[:, q], want_emb=False, k=5)
            assert torch.equal(out["sim"][:, q], one["sim"]), q
            assert torch.equal(out["topi"][:, q], one["topi"]), q
            assert torch.equal(out["topv"][:, q], one["topv"]), q
    finally:
        u.set_metric("l2")


@pytest.fixture(scope="module")
def grid26_oracle(seeded_state_dict, golden_dir):
    """oracle templates of grid26_b2 (the CPU restatement of the reference, run here) and the reference's
    broadcasting retrieval of the Q queries of each reference against them"""
    from oracle import unet_oracle as orc
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    unet_sd = {k: v for k, v in seeded_state_dict.items() if not k.startswith("encoder.")}
    rf, poses = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"])
    qs = multi_queries(g)
    with torch.no_grad():
        emb = orc.generate_templates(unet_sd, rf, poses)
    # retrieval(query [Q], template_feat [1, N]) per reference: query[:, None] - templates broadcasts to [Q, N]
    sim = torch.stack([orc.l2_similarity(qs[b], emb[b:b + 1]) for b in range(rf.shape[0])])
    return g, qs, sim


@pytest.mark.parametrize("mode", ["fp16", "parity"])
def test_multi_query_against_oracle(gpu_model, gpu_model_parity, grid26_oracle, mode):
    from oracle import unet_oracle as orc
    g, qs, sim_o = grid26_oracle
    m = gpu_model if mode == "fp16" else gpu_model_parity
    out = m.u_net.sweep(torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"]), query_feat=qs,
                        want_emb=False, k=5)
    e = max_rel(out["sim"], sim_o)
    idx_o = orc.topk_lowest_index(sim_o.reshape(-1, 26), 5).view(2, 5, 5)
    log("multi_query_oracle", mode=mode, sim_max_rel=e, topi=out["topi"].tolist(), ref=idx_o.tolist())
    assert e < SIM_TOL
    assert torch.equal(out["topi"].cpu(), idx_o)


def test_standalone_retrieval_broadcasts(gpu_model, golden_dir):
    from nope_b200.model import score_topk
    from oracle import unet_oracle as orc
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    rf, poses = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"])
    qs = multi_queries(g)
    emb = gpu_model.u_net.sweep(rf, poses, want_emb=True)["emb"]          # [2, 26, 8, 32, 32] fp32
    t1 = emb[:1]
    q = qs[0].cuda()                                                        # [5, 8, 32, 32]
    sim, idx = score_topk(q, t1, k=5)
    ref = orc.l2_similarity(q.cpu(), t1.cpu())                              # broadcast [5,1,...] - [1,26,...]
    e = max_rel(sim, ref)
    log("retrieval_broadcast", q_by_1=e)
    assert sim.shape == (5, 26) and idx.shape == (5, 5) and e < 1e-6
    assert torch.equal(idx.cpu(), orc.topk_lowest_index(sim.cpu(), 5))
    # one query against two template sets: [1] x [2, N] -> [2, N]
    sim2, _ = score_topk(q[:1], emb, k=5)
    ref2 = orc.l2_similarity(q[:1].cpu(), emb.cpu())
    assert sim2.shape == (2, 26) and max_rel(sim2, ref2) < 1e-6
    # equal batches: as before
    sim3, _ = score_topk(qs[:, 0].cuda(), emb, k=5)
    assert sim3.shape == (2, 26) and max_rel(sim3, orc.l2_similarity(qs[:, 0], emb.cpu())) < 1e-6
    with pytest.raises(ValueError):
        score_topk(qs[0, :3].cuda(), emb, k=5)
    # every metric: row q of a [Q] x [1, N] call equals the one-query call bit for bit
    for metric in METRICS:
        s, _ = score_topk(q, t1, k=5, metric=metric, threshold=0.2)
        for j in range(q.shape[0]):
            s1, _ = score_topk(q[j:j + 1], t1, k=5, metric=metric, threshold=0.2)
            assert torch.equal(s[j], s1[0]), (metric, j)
    # through the task module, on images
    from oracle import inputs
    imgs, _ = inputs.make_images(seed=3, batch=3)
    s_r, i_r = gpu_model.retrieval(imgs, t1)
    feats = gpu_model.u_net.encoder.encode_image(imgs.cuda())
    assert s_r.shape == (3, 26) and max_rel(s_r, orc.l2_similarity(feats.cpu(), t1.cpu())) < 1e-6


def test_predict_pose_multi_query_forms(gpu_model, golden_dir):
    from oracle import inputs
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    poses = torch.from_numpy(g["all_relativeR"])
    tposes = torch.from_numpy(g["template_poses"])
    q, r = inputs.make_images(seed=0, batch=2)
    q2, _ = inputs.make_images(seed=5, batch=2)
    q3, _ = inputs.make_images(seed=9, batch=2)
    qs = torch.stack([q, q2, q3], dim=1)                                    # [2, 3, 3, 256, 256]
    R, idx, sim = gpu_model.predict_pose(qs, r, poses, tposes, k=5)
    assert R.shape == (2, 3, 5, 3, 3) and idx.shape == (2, 3, 5) and sim.shape == (2, 3, 26)
    for j in range(3):
        R1, i1, s1 = gpu_model.predict_pose(qs[:, j], r, poses, tposes, k=5)
        assert torch.equal(idx[:, j], i1), j
        assert max_rel(sim[:, j], s1) < 1e-6, j
    assert torch.equal(R.cpu(), tposes[idx.cpu()])
    # broadcast form: one reference, queries [Q, 3, H, W]
    qb = qs[0]                                                              # the three queries of reference 0
    Rb, ib, sb = gpu_model.predict_pose(qb, r[:1], poses[:1], tposes, k=5)
    assert Rb.shape == (3, 5, 3, 3) and ib.shape == (3, 5) and sb.shape == (3, 26)
    for j in range(3):
        _, i1, s1 = gpu_model.predict_pose(qb[j:j + 1], r[:1], poses[:1], tposes, k=5)
        assert torch.equal(ib[j], i1[0]) and max_rel(sb[j], s1[0]) < 1e-6, j
    assert torch.equal(Rb.cpu(), tposes[ib.cpu()])


def test_ldm_multi_query_fused_scores_match_standalone(golden_dir):
    """LDM variant, 642 poses at chunk 256, Q = 4: the fused l2 scores equal a standalone scoring of the templates
    the same call wrote, and each query's scores and top-k equal a one-query sweep of that query bit for bit."""
    from nope_b200.ldm import UNetModelPose
    from nope_b200.model import score_topk
    from nope_b200.synth_weights import make_ldm_state_dict
    from oracle import unet_oracle as orc
    g = np.load(f"{golden_dir}/level2_642_b1.npz")
    poses = torch.from_numpy(g["all_relativeR"])
    gen = torch.Generator().manual_seed(4)
    ref = torch.randn(1, 4, 32, 32, generator=gen)
    qry = torch.randn(1, 4, 4, 32, 32, generator=gen)
    m = UNetModelPose(device="cuda:0", chunk=256).load_state_dict(make_ldm_state_dict(seed=0))
    out = m.sweep(ref, poses, qry, want_emb=True, k=5)
    assert out["sim"].shape == (1, 4, 642) and out["topi"].shape == (1, 4, 5)
    sim_s, idx_s = score_topk(qry[0].cuda(), out["emb"], k=5)
    e = max_rel(out["sim"][0], sim_s)
    log("ldm_multi_query", vs_standalone=e)
    assert e < 1e-5
    assert torch.equal(out["topi"][0].cpu(), orc.topk_lowest_index(out["sim"][0].cpu(), 5))
    for q in range(qry.shape[1]):
        one = m.sweep(ref, poses, qry[:, q], want_emb=True, k=5)
        assert torch.equal(one["emb"], out["emb"]), q
        assert torch.equal(one["sim"], out["sim"][:, q]), q
        assert torch.equal(one["topv"], out["topv"][:, q]), q
        assert torch.equal(one["topi"], out["topi"][:, q]), q
    # the latent-space predict_pose takes the same forms
    tp = torch.eye(3).expand(642, 3, 3).contiguous()
    R, idx, sim = m.predict_pose(qry[0], ref, poses, tp, k=5)
    assert R.shape == (4, 5, 3, 3) and idx.shape == (4, 5) and sim.shape == (4, 642)
    # as in PoseConditional.predict_pose: k > N is clamped to N, and template_poses [B, N, 3, 3] are read at row 0
    R4, idx4, sim4 = m.predict_pose(qry[0], ref, poses[:, :4], tp[:4], k=4)
    R5, idx5, sim5 = m.predict_pose(qry[0], ref, poses[:, :4], tp[:4], k=5)
    assert idx5.shape == (4, 4) and torch.equal(idx5, idx4) and torch.equal(sim5, sim4) and torch.equal(R5, R4)
    refs = torch.cat([ref, torch.randn(1, 4, 32, 32, generator=gen)])
    tp2 = torch.randn(2, 40, 3, 3, generator=gen)                           # a different grid per reference
    R2, idx2, _ = m.predict_pose(qry[0, :2], refs, poses[:, :40].expand(2, 40, 6), tp2, k=5)
    assert torch.equal(R2, tp2[0].cuda()[idx2]) and not torch.equal(R2[1], tp2[1].cuda()[idx2[1]])
    # a preallocated output that does not fit is refused, as by UNet.sweep
    with pytest.raises(ValueError):
        m.sweep(ref, poses, qry, want_emb=False, k=5, out={"sim": torch.empty((1, 4, 641), device="cuda:0")})
    del m


def test_caller_workspace_sized_for_one_query(seeded_state_dict, golden_dir):
    """a caller-owned workspace sized for Q = 1 refuses a Q = 4 sweep with a clear message; sized for B*Q*N
    scored triples it runs"""
    from nope_b200 import _lib
    from nope_b200.model import build_model
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    dev = torch.device("cuda:0")
    rf = torch.from_numpy(g["ref_feat"]).to(dev)
    poses = torch.from_numpy(g["all_relativeR"]).to(dev)
    qs = multi_queries(g, Q=4).to(dev)
    B, Q, N = 2, 4, 26
    m = build_model(device="cuda:0").load_state_dict(seeded_state_dict)
    u = m.u_net
    lib = _lib.load()
    sim = torch.empty((B, Q, N), device=dev)
    topv = torch.empty((B, Q, 5), device=dev)
    topi = torch.empty((B, Q, 5), device=dev, dtype=torch.int64)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def run():
        return lib.nope_unet_sweep_multi(u._handle(), _lib.ptr(rf), _lib.ptr(poses), B, N, _lib.ptr(qs), Q, None,
                                         _lib.ptr(sim), 5, _lib.ptr(topv), _lib.ptr(topi), 0, st)

    u.reserve(B * N, B, B * N)                 # sized for one query per reference
    assert run() != 0
    msg = lib.nope_last_error().decode()
    assert "workspace" in msg, msg
    u.reserve(B * N, B, B * Q * N)
    _lib.check(run())
    ref = u.sweep(rf, poses, query_feat=qs, want_emb=False, k=5)
    assert torch.equal(ref["sim"], sim) and torch.equal(ref["topi"], topi)
    # preallocated outputs that do not fit are refused with ValueError, as by UNetModelPose.sweep
    for out in ({"sim": sim[:, :1]}, {"sim": sim.transpose(1, 2).contiguous().transpose(1, 2)},
                {"topv": topv, "topi": topi.to(torch.int32)}):
        with pytest.raises(ValueError):
            u.sweep(rf, poses, query_feat=qs, want_emb=False, k=5, out=out)
    del m
