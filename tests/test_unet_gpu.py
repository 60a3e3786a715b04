"""GPU: the whole hot path through the public Python surface (which calls the C ABI)
against (a) the golden fixtures generated from the unmodified reference and (b) the
oracle run live on the host CPU.

Tolerances (fp16 storage, fp32 accumulation/statistics; SURVEY.md section 7 measured
1.1e-3 / 1.7e-4 for fp16 autocast of the reference itself):
  embeddings  rel-L2 <= EMB_TOL, similarity rel <= SIM_TOL, top-1 index identical,
  top-5 set identical where the reference's own adjacent score gaps exceed 2*SIM_TOL."""
import numpy as np
import pytest
import torch

from _util import log, max_rel, rel_l2

pytestmark = pytest.mark.gpu

# Stated tolerances (BASELINE.json north_star: embeddings and scores within 1e-3 of the fp32 reference,
# argmax identical):
#   precision "parity" (split precision)  embeddings <= 1e-3 (measured ~1e-4), scores <= 1e-3, top-5 identical
#   precision "fp16"  (default, fast)     scores <= 1e-3 (measured 7e-4) and argmax identical, but embeddings
#                                         1.2-1.5e-3: fp16 WEIGHT rounding alone is 0.9e-3 and every stored
#                                         activation adds 2.8e-4 rms (tools/precision_sim.py) -- the fast mode
#                                         is gated at 2e-3 and does NOT claim the embedding bar
EMB_TOL = 2.0e-3
EMB_TOL_PARITY = 1e-3
SIM_TOL = 1e-3


def _swaps(idx_ref, idx):
    """positions 2..5 of the top-5 that differ from the reference (position 1 is asserted equal)"""
    idx_ref = torch.as_tensor(idx_ref)
    return int((idx.cpu()[:, 1:] != idx_ref[:, 1:]).sum())


def _cmp_ranking(sim_ref, idx_ref, idx, tol):
    """top-1 must match; later ranks must match unless the reference scores of the two
    candidates are closer than tol (relative)."""
    sim_ref = torch.as_tensor(sim_ref)
    idx_ref = torch.as_tensor(idx_ref)
    assert torch.equal(idx[:, 0].cpu(), idx_ref[:, 0]), (idx, idx_ref)
    for b in range(idx_ref.shape[0]):
        for r in range(idx_ref.shape[1]):
            i, j = int(idx[b, r]), int(idx_ref[b, r])
            if i != j:
                gap = abs(float(sim_ref[b, i] - sim_ref[b, j])) / abs(float(sim_ref[b, j]))
                assert gap < 2 * tol, (b, r, i, j, gap)


def test_cfg1_golden(gpu_model, golden_dir):
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    rf = torch.from_numpy(g["ref_feat"])
    qf = torch.from_numpy(g["query_feat"])
    poses = torch.from_numpy(g["all_relativeR"])
    out = gpu_model.u_net.sweep(rf, poses, query_feat=qf, want_emb=True, k=5)
    e_emb = rel_l2(out["emb"], torch.from_numpy(g["emb"]))
    e_sim = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
    log("cfg1_golden", emb_rel_l2=e_emb, sim_max_rel=e_sim, topi=out["topi"].tolist(),
        ref_topi=g["nearest_idx"].tolist(), launches=gpu_model.u_net.last_launch_count)
    assert e_emb < EMB_TOL and e_sim < SIM_TOL
    _cmp_ranking(g["similarity"], g["nearest_idx"], out["topi"], SIM_TOL)


def test_cfg1_end_to_end_from_images(gpu_model, golden_dir):
    """images -> encoder (torch/cuDNN fp32) -> sweep -> fused score/top-k, via predict_pose"""
    from oracle import inputs
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    q, r = inputs.make_images(seed=0, batch=1)
    poses = torch.from_numpy(g["all_relativeR"])
    tposes = torch.from_numpy(g["template_poses"])
    R, idx, sim, emb = gpu_model.predict_pose(q, r, poses, tposes, k=5, return_templates=True)
    e_q = rel_l2(gpu_model.u_net.encoder.encode_image(q), torch.from_numpy(g["query_feat"]))
    e_emb = rel_l2(emb, torch.from_numpy(g["emb"]))
    e_sim = max_rel(sim, torch.from_numpy(g["similarity"]))
    log("cfg1_e2e", enc_rel_l2=e_q, emb_rel_l2=e_emb, sim_max_rel=e_sim)
    assert e_q < 1e-4 and e_emb < EMB_TOL and e_sim < SIM_TOL
    assert R.shape == (1, 5, 3, 3)
    assert torch.equal(R[0, 0].cpu(), tposes[int(g["nearest_idx"][0, 0])])
    # the reference's own surface: generate_templates + retrieval
    # (its encoder runs at batch 1 instead of predict_pose's batch 2: cuDNN may pick another
    # algorithm, so latents differ at the 1e-6 level and fp16 re-rounding amplifies that)
    emb2, _, _ = gpu_model.generate_templates(r, poses, None)
    sim2, idx2 = gpu_model.retrieval(q, emb2)
    assert torch.equal(idx2, idx) and rel_l2(sim2, sim) < 5e-4
    assert rel_l2(emb2, emb) < EMB_TOL
    # determinism: the same call twice is bit-identical (no atomics in any reduction)
    R3, idx3, sim3, emb3 = gpu_model.predict_pose(q, r, poses, tposes, k=5, return_templates=True)
    assert torch.equal(emb3, emb) and torch.equal(sim3, sim) and torch.equal(idx3, idx)


def test_grid26_b2_golden(gpu_model, golden_dir):
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    rf, qf = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["query_feat"])
    poses = torch.from_numpy(g["all_relativeR"])
    out = gpu_model.u_net.sweep(rf, poses, query_feat=qf, want_emb=True, k=5)
    emb = out["emb"].cpu()
    e0 = rel_l2(emb[0, 0], torch.from_numpy(g["emb_b0_n0"]))
    e1 = rel_l2(emb[1, 25], torch.from_numpy(g["emb_b1_n25"]))
    e_l2 = max_rel(emb.flatten(2).norm(dim=2), torch.from_numpy(g["emb_l2"]))
    e_sim = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
    log("grid26_golden", emb00=e0, emb125=e1, emb_l2=e_l2, sim_max_rel=e_sim,
        topi=out["topi"].tolist(), ref=g["nearest_idx"].tolist())
    assert max(e0, e1) < EMB_TOL and e_sim < SIM_TOL
    _cmp_ranking(g["similarity"], g["nearest_idx"], out["topi"], SIM_TOL)
    # chunking must not change anything: 7 hypotheses per chunk vs one chunk
    gpu_model.u_net.set_chunk(7)
    out2 = gpu_model.u_net.sweep(rf, poses, query_feat=qf, want_emb=True, k=5)
    gpu_model.u_net.set_chunk(642)
    assert torch.equal(out2["emb"], out["emb"]) and torch.equal(out2["topi"], out["topi"])
    assert torch.equal(out2["sim"], out["sim"])


def test_layer_taps_vs_live_oracle(gpu_model, seeded_state_dict, golden_dir):
    """per-layer activations of one sweep against the oracle (CPU, run here)."""
    from oracle import unet_oracle as orc
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    unet_sd = {k: v for k, v in seeded_state_dict.items() if not k.startswith("encoder.")}
    rf = torch.from_numpy(g["ref_feat"])
    poses = torch.from_numpy(g["all_relativeR"])[0, :3]
    taps = {}
    with torch.no_grad():
        orc.unet_forward(unet_sd, rf.expand(3, -1, -1, -1), poses, taps=taps)
    worst = 0.0
    for name in ["init_conv", "downs.0.0", "downs.0.1", "downs.0.2", "downs.0.3", "downs.1.2",
                 "downs.2.3", "downs.3.3", "mid.0", "mid.1", "ups.0.0", "ups.0.3", "ups.1.3",
                 "ups.2.3", "ups.3.3", "final_res_block", "final_conv.0"]:
        got = gpu_model.u_net.debug_tap(rf, poses, name)
        e = rel_l2(got, taps[name])
        worst = max(worst, e)
        log("tap", layer=name, rel_l2=e)
    assert worst < EMB_TOL


def test_forward_call_and_loss(gpu_model, golden_dir):
    """UNet.__call__(x, pose) and PoseConditional.forward (loss) keep the reference surface."""
    from oracle import inputs
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    rf = torch.from_numpy(g["ref_feat"])
    y = gpu_model.u_net(rf, torch.from_numpy(g["all_relativeR"][:, 2]))
    assert y.shape == (1, 8, 32, 32)
    assert rel_l2(y, torch.from_numpy(g["emb"][:, 2])) < EMB_TOL
    q, r = inputs.make_images(seed=0, batch=1)
    loss = gpu_model.forward(q, r, torch.from_numpy(g["all_relativeR"][:, 2]))
    ref_loss = (torch.from_numpy(g["emb"][:, 2]) - torch.from_numpy(g["query_feat"])).abs().mean()
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * float(ref_loss)


@pytest.mark.parametrize("metric", ["cosine", "cosine_occlusion"])
def test_fused_extension_metrics(gpu_model, golden_dir, metric):
    """SURVEY 8 row f4: the cosine / occlusion-aware similarities are evaluated in the sweep's last
    layer (no [B,N,C,32,32] tensor) and must equal (a) the standalone scoring of the materialised
    templates and (b) the torch oracle of the metric on those templates."""
    from nope_b200.model import score_topk
    from oracle import unet_oracle as orc
    g = np.load(f"{golden_dir}/grid26_b2.npz")
    rf, qf = torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["query_feat"])
    poses = torch.from_numpy(g["all_relativeR"])
    u = gpu_model.u_net
    try:
        u.set_metric(metric, 0.2)
        out = u.sweep(rf, poses, query_feat=qf, want_emb=True, k=5)
    finally:
        u.set_metric("l2")
    sim2, idx2 = score_topk(qf.cuda(), out["emb"], k=5, metric=metric, threshold=0.2)
    fn = orc.cosine_similarity if metric == "cosine" else orc.cosine_occlusion_similarity
    ref = fn(qf, out["emb"].cpu())
    e_std, e_orc = max_rel(out["sim"], sim2), max_rel(out["sim"], ref)
    log("fused_metric", metric=metric, vs_standalone=e_std, vs_oracle=e_orc, topi=out["topi"].tolist())
    assert e_std < 1e-5 and e_orc < 1e-5
    assert torch.equal(out["topi"].cpu(), orc.topk_lowest_index(out["sim"].cpu(), 5))
    # through the task module: similarity_metric in testing_config (configs/model/template_base.yaml:24)
    from oracle import inputs
    q, r = inputs.make_images(seed=0, batch=2)
    old = gpu_model.testing_config.similarity_metric
    try:
        gpu_model.testing_config.similarity_metric = metric
        _, idx3, sim3 = gpu_model.predict_pose(q, r, poses, None, k=5)
    finally:
        gpu_model.testing_config.similarity_metric = old
        u.set_metric("l2")
    assert sim3.shape == (2, 26) and idx3.shape == (2, 5)
    assert torch.equal(idx3.cpu(), orc.topk_lowest_index(sim3.cpu(), 5))


def test_parity_mode_meets_the_north_star_tolerance(gpu_model_parity, gpu_model, golden_dir):
    """precision="parity": every convolution runs A_hi W_hi + A_hi W_lo + A_lo W_hi on fp16 (hi, lo) pairs
    (22 significant bits), activations travel as pairs.  Against the UNMODIFIED reference's goldens:
    embeddings <= 1e-3 (the stated bar, with an order of magnitude to spare), scores <= 1e-3, the whole
    top-5 identical; the fast fp16 mode's rank swaps on the same grids are reported next to it."""
    m = gpu_model_parity
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    out = m.u_net.sweep(torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"]),
                        query_feat=torch.from_numpy(g["query_feat"]), want_emb=True, k=5)
    e1 = rel_l2(out["emb"], torch.from_numpy(g["emb"]))
    s1 = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
    assert e1 < EMB_TOL_PARITY and s1 < SIM_TOL
    assert torch.equal(out["topi"].cpu(), torch.from_numpy(g["nearest_idx"]))
    g2 = np.load(f"{golden_dir}/grid26_b2.npz")
    out2 = m.u_net.sweep(torch.from_numpy(g2["ref_feat"]), torch.from_numpy(g2["all_relativeR"]),
                         query_feat=torch.from_numpy(g2["query_feat"]), want_emb=True, k=5)
    e2 = max(rel_l2(out2["emb"][0, 0], torch.from_numpy(g2["emb_b0_n0"])),
             rel_l2(out2["emb"][1, 25], torch.from_numpy(g2["emb_b1_n25"])))
    s2 = max_rel(out2["sim"], torch.from_numpy(g2["similarity"]))
    assert e2 < EMB_TOL_PARITY and s2 < SIM_TOL
    assert torch.equal(out2["topi"].cpu(), torch.from_numpy(g2["nearest_idx"]))
    g3 = np.load(f"{golden_dir}/level2_642_b1.npz")
    args3 = (torch.from_numpy(g3["ref_feat"]), torch.from_numpy(g3["all_relativeR"]))
    out3 = m.u_net.sweep(*args3, query_feat=torch.from_numpy(g3["query_feat"]), want_emb=True, k=5)
    e3 = max(rel_l2(out3["emb"][0, 0], torch.from_numpy(g3["emb_n0"])),
             rel_l2(out3["emb"][0, 641], torch.from_numpy(g3["emb_n641"])))
    s3 = max_rel(out3["sim"], torch.from_numpy(g3["similarity"]))
    fast = gpu_model.u_net.sweep(*args3, query_feat=torch.from_numpy(g3["query_feat"]), want_emb=False, k=5)
    log("parity_mode", cfg1_emb=e1, cfg1_sim=s1, grid26_emb=e2, grid26_sim=s2, level2_642_emb=e3, level2_642_sim=s3,
        top5_642=out3["topi"].tolist(), swaps_642_parity=_swaps(g3["nearest_idx"], out3["topi"]),
        swaps_642_fp16=_swaps(g3["nearest_idx"], fast["topi"]))
    assert e3 < EMB_TOL_PARITY and s3 < SIM_TOL
    assert torch.equal(out3["topi"].cpu(), torch.from_numpy(g3["nearest_idx"]))
    # chunking / determinism hold in this mode too
    m.u_net.set_chunk(100)
    out4 = m.u_net.sweep(*args3, query_feat=torch.from_numpy(g3["query_feat"]), want_emb=False, k=5)
    m.u_net.set_chunk(642)
    assert torch.equal(out4["sim"], out3["sim"]) and torch.equal(out4["topi"], out3["topi"])


def test_parity_fast_mode_meets_the_north_star_tolerance(seeded_state_dict, golden_dir):
    """precision="parity_fast": (hi, lo) pairs on the residual stream, skips and resampled maps, a single fp16 inside
    each ResnetBlock (block2 runs two products per tap).  Budget from tools/precision_sim.py: 4.3e-4 from those tensors
    on top of the parity mode's 2.2e-4; gated at the same north-star 1e-3 on embeddings and scores, top-5 identical."""
    from nope_b200.model import build_model
    m = build_model(device="cuda:0", precision="parity_fast")
    m.load_state_dict(seeded_state_dict)
    g = np.load(f"{golden_dir}/cfg1_b1_n6.npz")
    out = m.u_net.sweep(torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"]),
                        query_feat=torch.from_numpy(g["query_feat"]), want_emb=True, k=5)
    e1 = rel_l2(out["emb"], torch.from_numpy(g["emb"]))
    s1 = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
    g3 = np.load(f"{golden_dir}/level2_642_b1.npz")
    out3 = m.u_net.sweep(torch.from_numpy(g3["ref_feat"]), torch.from_numpy(g3["all_relativeR"]),
                         query_feat=torch.from_numpy(g3["query_feat"]), want_emb=True, k=5)
    e3 = max(rel_l2(out3["emb"][0, 0], torch.from_numpy(g3["emb_n0"])),
             rel_l2(out3["emb"][0, 641], torch.from_numpy(g3["emb_n641"])))
    s3 = max_rel(out3["sim"], torch.from_numpy(g3["similarity"]))
    log("parity_fast_mode", cfg1_emb=e1, cfg1_sim=s1, level2_642_emb=e3, level2_642_sim=s3,
        swaps_642=_swaps(g3["nearest_idx"], out3["topi"]), launches=m.u_net.last_launch_count)
    assert e1 < EMB_TOL_PARITY and s1 < SIM_TOL and e3 < EMB_TOL_PARITY and s3 < SIM_TOL
    assert torch.equal(out["topi"].cpu(), torch.from_numpy(g["nearest_idx"]))
    assert torch.equal(out3["topi"].cpu(), torch.from_numpy(g3["nearest_idx"]))


def test_exact_weights_mode(seeded_state_dict, golden_dir):
    """precision="fp16_w2" (W_hi + W_lo K-segments, fp16 activations): measured between the two other
    modes; gated at the fast mode's tolerance."""
    from nope_b200.model import build_model
    m = build_model(device="cuda:0", precision="fp16_w2")
    m.load_state_dict(seeded_state_dict)
    g3 = np.load(f"{golden_dir}/level2_642_b1.npz")
    out = m.u_net.sweep(torch.from_numpy(g3["ref_feat"]), torch.from_numpy(g3["all_relativeR"]),
                        query_feat=torch.from_numpy(g3["query_feat"]), want_emb=True, k=5)
    e = max(rel_l2(out["emb"][0, 0], torch.from_numpy(g3["emb_n0"])), rel_l2(out["emb"][0, 641], torch.from_numpy(g3["emb_n641"])))
    s = max_rel(out["sim"], torch.from_numpy(g3["similarity"]))
    log("w2_mode", level2_642_emb=e, level2_642_sim=s, swaps=_swaps(g3["nearest_idx"], out["topi"]))
    assert e < EMB_TOL and s < SIM_TOL
    assert int(out["topi"][0, 0]) == int(g3["nearest_idx"][0, 0])


def test_bf16_storage_mode(seeded_state_dict, golden_dir):
    """precision="bf16" (BASELINE configs[2]): bf16 weights and activations, fp32 accumulation / statistics.
    Stated tolerance: embeddings 2e-2 rel-L2 and scores 1.5e-2 of the fp32 reference (measured 1.0e-2 / 7e-3;
    the reference under bf16 autocast is itself 8.8e-3 / 1.5e-3, SURVEY.md section 7), and the best pose must
    be one the reference scores within 1.5e-2 of its own best -- bf16 cannot separate closer candidates."""
    from nope_b200.model import build_model
    m = build_model(device="cuda:0", precision="bf16")
    m.load_state_dict(seeded_state_dict)
    for name, keys in (("cfg1_b1_n6", None), ("level2_642_b1", ("emb_n0", 0, 0))):
        g = np.load(f"{golden_dir}/{name}.npz")
        out = m.u_net.sweep(torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"]),
                            query_feat=torch.from_numpy(g["query_feat"]), want_emb=True, k=5)
        e = rel_l2(out["emb"], torch.from_numpy(g["emb"])) if keys is None else \
            rel_l2(out["emb"][0, 0], torch.from_numpy(g["emb_n0"]))
        s = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
        s_ref = torch.from_numpy(g["similarity"])
        best = int(out["topi"][0, 0])
        margin = float(s_ref[0].max() - s_ref[0, best]) / abs(float(s_ref[0].max()))
        log("bf16_mode", fixture=name, emb_rel_l2=e, sim_max_rel=s, top1=best, ref_top1=int(g["nearest_idx"][0, 0]),
            ref_margin_of_our_top1=margin)
        assert e < 2e-2 and s < 1.5e-2 and margin < 1.5e-2
    again = m.u_net.sweep(torch.from_numpy(g["ref_feat"]), torch.from_numpy(g["all_relativeR"]),
                          query_feat=torch.from_numpy(g["query_feat"]), want_emb=False, k=5)
    assert torch.equal(again["sim"], out["sim"])                      # deterministic


def test_bad_arguments_raise(gpu_model):
    from nope_b200 import NopeError
    rf = torch.zeros(1, 8, 32, 32)
    with pytest.raises(NopeError):
        gpu_model.u_net.sweep(rf, torch.zeros(1, 3, 6), query_feat=rf, k=5)   # k > N


def test_full_size_grid_properties(gpu_model):
    """BASELINE configs[1] size (642-pose grid, one query): size-independent properties instead
    of an oracle run (642 CPU forwards would take minutes):
      * determinism: the same sweep twice is bit-identical;
      * pose-permutation equivariance: permuting the grid permutes the scores, bit for bit
        (every hypothesis is an independent forward, whatever tile / cluster it lands in);
      * duplicated poses give identical scores and the top-k tie-break picks the lower index;
      * chunk-size invariance at a size with ragged last tiles (642 = 5*128 + 2)."""
    from nope_b200.poses import synthetic_pose_batch
    g = torch.Generator().manual_seed(7)
    rf = torch.randn(1, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn(1, 8, 32, 32, generator=g) * 1.5
    poses, _ = synthetic_pose_batch(642, 1)
    u = gpu_model.u_net
    a = u.sweep(rf, poses, query_feat=qf, want_emb=False, k=5)
    b = u.sweep(rf, poses, query_feat=qf, want_emb=False, k=5)
    assert torch.equal(a["sim"], b["sim"]) and torch.equal(a["topi"], b["topi"])
    perm = torch.randperm(642, generator=g)
    c = u.sweep(rf, poses[:, perm], query_feat=qf, want_emb=False, k=5)
    assert torch.equal(c["sim"].cpu(), a["sim"].cpu()[:, perm])
    assert torch.equal(perm[c["topi"].cpu()[0]], a["topi"].cpu()[0])
    dup = poses.clone()
    best = int(a["topi"][0, 0])
    other = 600 if best != 600 else 601
    dup[0, other] = dup[0, best]
    d = u.sweep(rf, dup, query_feat=qf, want_emb=False, k=5)
    assert d["sim"][0, other] == d["sim"][0, best]
    assert d["topi"][0, :2].tolist() == sorted([best, other])
    u.set_chunk(100)
    e = u.sweep(rf, poses, query_feat=qf, want_emb=False, k=5)
    u.set_chunk(642)
    assert torch.equal(e["sim"], a["sim"]) and torch.equal(e["topi"], a["topi"])
    log("full_grid_642", top5=a["topi"].tolist(), launches=u.last_launch_count)


def test_batch_of_queries_is_independent(gpu_model):
    """configs[2] shape in miniature (B=3 queries x 162-pose grid): each batch row equals the
    same query run alone (hypotheses of different references never interact)."""
    from nope_b200.poses import synthetic_pose_batch
    g = torch.Generator().manual_seed(9)
    rf = torch.randn(3, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn(3, 8, 32, 32, generator=g) * 1.5
    poses, _ = synthetic_pose_batch(162, 3)
    u = gpu_model.u_net
    full = u.sweep(rf, poses, query_feat=qf, want_emb=True, k=5)
    for b in range(3):
        one = u.sweep(rf[b:b + 1], poses[b:b + 1], query_feat=qf[b:b + 1], want_emb=True, k=5)
        assert torch.equal(one["sim"][0], full["sim"][b])
        assert torch.equal(one["topi"][0], full["topi"][b])
        assert torch.equal(one["emb"][0], full["emb"][b])


def test_shard_size_invariance(gpu_model):
    """What the multi-GPU path relies on: sweeping a slice of the pose grid gives bit-identical
    scores to the same poses inside the full sweep, for any slice size (the launch size changes
    tile composition and CTA counts, never a reduction order)."""
    from nope_b200.poses import synthetic_pose_batch
    g = torch.Generator().manual_seed(11)
    rf = torch.randn(2, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn(2, 8, 32, 32, generator=g) * 1.5
    poses, _ = synthetic_pose_batch(162, 2)
    u = gpu_model.u_net
    full = u.sweep(rf, poses, query_feat=qf, want_emb=False, k=5)
    for lo, hi in [(0, 81), (81, 162), (0, 1), (5, 162), (100, 103)]:
        part = u.sweep(rf, poses[:, lo:hi].contiguous(), query_feat=qf, want_emb=False,
                       k=min(5, hi - lo), idx_base=lo)
        assert torch.equal(part["sim"], full["sim"][:, lo:hi]), (lo, hi)
        assert int(part["topi"].min()) >= lo and int(part["topi"].max()) < hi


def test_native_encoder_matches_oracle_and_torch(gpu_model, seeded_state_dict):
    """template encoder on the wgmma kernel with split-precision operands (SURVEY 8 row f1)
    vs the oracle's torch-CPU fp32 restatement and vs the cuDNN fp32 module: fp32-level parity
    (the latents feed the score directly; TF32 / fp16 would be 2-3e-3 off)."""
    from oracle import inputs, unet_oracle as orc
    from nope_b200.encoder import FeatureExtractor
    enc_sd = {k[len("encoder."):]: v for k, v in seeded_state_dict.items() if k.startswith("encoder.")}
    q, r = inputs.make_images(seed=5, batch=2)
    x = torch.cat([q, r])[:3]                       # batch 3: odd tile counts at every level
    with torch.no_grad():
        ref = orc.encode_image(enc_sd, x)
    enc = gpu_model.u_net.encoder
    assert enc.backend in ("auto", "b200")
    got = enc.encode_image(x)
    e = rel_l2(got, ref)
    m = max_rel(got, ref)
    fe_t = FeatureExtractor(descriptor_size=8, backend="torch").cuda()
    fe_t.load_state_dict({k: v for k, v in enc_sd.items()
                          if k.startswith("backbone.") or k.startswith("projector.")})
    e_t = rel_l2(fe_t.encode_image(x), ref)
    log("native_encoder", rel_l2=e, max_rel=m, cudnn_fp32_rel_l2=e_t)
    # measured 5e-5 (cuDNN fp32: 2e-6; cuDNN TF32 / fp16: 2e-3 / 3e-3): 22-bit operands, the
    # A_lo*W_lo term dropped, and the tensor core's non-IEEE fp32 accumulation over K <= 13824
    assert e < 1.5e-4 and m < 3e-4
    assert torch.equal(enc.encode_image(x), got)    # deterministic
    # any batch size: the engine walks the images 32 at a time (predict_pose concatenates query and reference
    # views, model.py:112, so an evaluation batch of 40 encodes 80 images in one call)
    big = x[:2].repeat(35, 1, 1, 1)                 # 70 images: two full chunks + a ragged one
    out = enc.encode_image(big)
    assert out.shape[0] == 70 and torch.equal(out[68:70], out[0:2]) and torch.equal(out[33], out[1])
    assert rel_l2(out[:2], ref[:2]) < 1.5e-4


def test_full_level2_grid_against_reference_golden(gpu_model, golden_dir):
    """BASELINE configs[1] at full size against the reference itself: 642-pose level-2 grid
    (the grid the reference ships), one query; fixture = the unmodified reference modules on CPU
    (tests/golden/level2_642_b1.npz, oracle/make_golden.py --only-full-grid)."""
    from oracle import inputs
    g = np.load(f"{golden_dir}/level2_642_b1.npz")
    poses = torch.from_numpy(g["all_relativeR"])
    # (a) from the reference's latents: UNet sweep + score only
    out = gpu_model.u_net.sweep(torch.from_numpy(g["ref_feat"]), poses,
                                query_feat=torch.from_numpy(g["query_feat"]), want_emb=True, k=5)
    e_sim = max_rel(out["sim"], torch.from_numpy(g["similarity"]))
    e0 = rel_l2(out["emb"][0, 0], torch.from_numpy(g["emb_n0"]))
    e1 = rel_l2(out["emb"][0, 641], torch.from_numpy(g["emb_n641"]))
    # (b) from the images, through the native encoder and the public predict_pose
    q, r = inputs.make_images(seed=2, batch=1)
    _, idx2, sim2 = gpu_model.predict_pose(q, r, poses, None, k=5)
    e_sim2 = max_rel(sim2, torch.from_numpy(g["similarity"]))
    log("level2_642_golden", sim_max_rel=e_sim, sim_max_rel_from_images=e_sim2, emb0=e0, emb641=e1,
        topi=out["topi"].tolist(), topi_from_images=idx2.tolist(), ref=g["nearest_idx"].tolist())
    assert e_sim < SIM_TOL and e_sim2 < SIM_TOL and max(e0, e1) < EMB_TOL
    _cmp_ranking(g["similarity"], g["nearest_idx"], out["topi"], SIM_TOL)
    _cmp_ranking(g["similarity"], g["nearest_idx"], idx2, SIM_TOL)


@pytest.mark.parametrize("dim", [64, 128])
def test_other_unet_widths_vs_live_oracle(dim):
    """UNet(u_net_dim=64 / 128) -- the widths the reference's own smoke block uses
    (u_net.py:201-217 builds u_net_dim=64): exercises the 64- and 128-channel N-tile variants of
    the convolution kernel through the whole pipeline, against the oracle run here on CPU."""
    from oracle import unet_oracle as orc, weights
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.unet import UNet
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sd = weights.make_unet_state_dict(seed=3, u_net_dim=dim)
    unet = UNet(u_net_dim=dim, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8),
                pose_mlp_name="single_layer", device="cuda:0")
    unet.load_state_dict(sd)
    g = torch.Generator().manual_seed(dim)
    rf = torch.randn(2, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn(2, 8, 32, 32, generator=g) * 1.5
    poses = torch.randn(2, 5, 6, generator=g)
    out = unet.sweep(rf, poses, query_feat=qf, want_emb=True, k=3)
    with torch.no_grad():
        emb = orc.generate_templates(sd, rf, poses)
        sim = orc.l2_similarity(qf, emb)
    e_emb, e_sim = rel_l2(out["emb"], emb), max_rel(out["sim"], sim)
    log("unet_width", dim=dim, emb_rel_l2=e_emb, sim_max_rel=e_sim)
    assert e_emb < EMB_TOL and e_sim < 2 * SIM_TOL
    assert torch.equal(out["topi"].cpu(), orc.topk_lowest_index(out["sim"].cpu(), 3))


@pytest.mark.parametrize("B,N,chunk", [(1, 1, 642), (1, 7, 3), (2, 9, 5), (3, 17, 642), (1, 131, 128),
                                       (2, 65, 64)])
def test_ragged_batches_equal_single_hypothesis_runs(gpu_model, B, N, chunk):
    """Every (reference, pose) forward is independent (model.py:212-222): for ragged sizes (partial
    128-pixel tiles at every resolution, odd CTA-pair counts, chunk tails of 1) the batched sweep
    must equal, bit for bit, the same hypothesis swept alone."""
    g = torch.Generator().manual_seed(B * 1000 + N)
    rf = torch.randn(B, 8, 32, 32, generator=g) * 1.5
    qf = torch.randn(B, 8, 32, 32, generator=g) * 1.5
    poses = torch.randn(B, N, 6, generator=g)
    u = gpu_model.u_net
    u.set_chunk(chunk)
    full = u.sweep(rf, poses, query_feat=qf, want_emb=True, k=min(5, N))
    u.set_chunk(642)
    picks = sorted({0, N - 1, N // 2, min(N - 1, chunk), max(0, chunk - 1) % N})
    for b in range(B):
        for n in picks:
            one = u.sweep(rf[b:b + 1], poses[b:b + 1, n:n + 1], query_feat=qf[b:b + 1], want_emb=True)
            assert torch.equal(one["emb"][0, 0], full["emb"][b, n]), (b, n)
            assert torch.equal(one["sim"][0, 0], full["sim"][b, n]), (b, n)
    assert torch.equal(full["topi"].cpu(),
                       __import__("oracle.unet_oracle", fromlist=["x"]).topk_lowest_index(full["sim"].cpu(), min(5, N)))
