"""GPU: the LDM-variant UNet (UNetModelPose, SURVEY.md 8 f2) through the Python mirror / C ABI
against the oracle run live on the host CPU and the golden fixture from the unmodified reference.

Every module is also driven in isolation (nope_ldm_run_block): it gets the ORACLE's input for
that module and must reproduce the oracle's output, so one failing kernel does not hide the rest.

Tolerances (fp16 storage of activations / weights / softmax probabilities, fp32 accumulation,
statistics, softmax and LayerNorm): per module rel-L2 <= BLOCK_TOL; l2 scores max-rel <= SIM_TOL;
whole network embeddings rel-L2 <= EMB_TOL = the north-star 1e-3 in the exact-weights mode
(precision="fp16_w2": W = W_hi + W_lo K-segments), <= EMB_TOL_FP16 in the fast fp16-weights mode, whose
weight rounding alone is 0.62e-3 of its measured 1.08e-3 (CPU experiment on the oracle, DESIGN.md)."""
import numpy as np
import pytest
import torch

from _util import log, max_rel, rel_l2

pytestmark = pytest.mark.gpu

BLOCK_TOL = 1e-3    # measured 3.0e-4 .. 4.1e-4 per module
EMB_TOL = 1e-3      # exact-weights mode: the north-star tolerance
EMB_TOL_FP16 = 1.5e-3   # fp16-weights mode: measured 1.07e-3 end to end (cumulative 1.3e-3 at the bottleneck)
SIM_TOL = 1e-3      # measured 2.9e-5
N_HYP = 2


def _plan():
    from nope_b200.synth_weights import ldm_block_plan
    return ldm_block_plan()


def _modules():
    """(name, kind, input tap(s), output tap) for every module of the forward pass."""
    inp, _, out = _plan()
    mods = []
    for i, b in enumerate(inp):
        p = f"input_blocks.{i}"
        prev = f"input_blocks.{i - 1}"
        if b[0] == "res":
            mods.append((p + ".0", "res", (prev, None), p + ".0"))
            mods.append((p + ".1", "st", (p + ".0", None), p))
        elif b[0] == "down":
            mods.append((p + ".0.op", "resample", (prev, None), p))
    last_in = f"input_blocks.{len(inp) - 1}"
    mods.append(("middle_block.0", "res", (last_in, None), "middle_block.0"))
    mods.append(("middle_block.1", "st", ("middle_block.0", None), "middle_block.1"))
    mods.append(("middle_block.2", "res", ("middle_block.1", None), "middle_block"))
    prev = "middle_block"
    for i, b in enumerate(out):
        p = f"output_blocks.{i}"
        mods.append((p + ".0", "res", (prev, f"input_blocks.{len(inp) - 1 - i}"), p + ".0"))
        mods.append((p + ".1", "st", (p + ".0", None), p + ".1"))
        if b[4]:
            mods.append((p + ".2.conv", "resample", (p + ".1", None), p))
        prev = p
    return mods


@pytest.fixture(scope="module")
def ldm_sd():
    from nope_b200.synth_weights import make_ldm_state_dict
    return make_ldm_state_dict(seed=0)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(f"{golden_dir}/ldm_b1_n3.npz")


@pytest.fixture(scope="module")
def oracle_taps(ldm_sd, golden):
    from oracle import ldm_oracle
    ref = torch.from_numpy(golden["ref_latent"])
    poses = torch.from_numpy(golden["all_relativeR"])[0, :N_HYP]
    taps = {}
    with torch.no_grad():
        emb = ldm_oracle.ldm_forward(ldm_sd, ref.expand(N_HYP, -1, -1, -1), poses, taps=taps)
    taps["emb"] = emb
    taps["poses"] = poses
    return taps


@pytest.fixture(scope="module")
def ldm_model(ldm_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.ldm import UNetModelPose
    m = UNetModelPose(device="cuda:0", chunk=8)
    m.load_state_dict(ldm_sd)
    return m


@pytest.mark.parametrize("n_tok,C", [(64, 1024), (256, 512), (1024, 256), (320, 64)])
def test_mh_attention(n_tok, C):
    """softmax(q k^T / sqrt(32)) v per head against torch fp32 on the fp16-rounded operands."""
    from nope_b200.ldm import mh_attention
    g = torch.Generator().manual_seed(n_tok + C)
    qkv = torch.randn(2, n_tok, 3 * C, generator=g) * 1.5
    qkv = qkv.half().float()
    out = mh_attention(qkv.cuda()).cpu()
    H = C // 32
    q, k, v = [t.reshape(2, n_tok, H, 32).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=-1)]
    att = (torch.einsum("bhid,bhjd->bhij", q, k) * 32 ** -0.5).softmax(dim=-1)
    ref = torch.einsum("bhij,bhjd->bhid", att, v).permute(0, 2, 1, 3).reshape(2, n_tok, C)
    e = rel_l2(out, ref)
    log("ldm_mh_attention", n_tok=n_tok, C=C, rel_l2=e, max_rel=max_rel(out, ref))
    assert e < 1.5e-3


@pytest.mark.parametrize("mod", _modules(), ids=lambda m: m[0])
def test_module_in_isolation(ldm_model, oracle_taps, mod):
    name, kind, (in0, in1), out_tap = mod
    x0 = oracle_taps[in0]
    x1 = oracle_taps[in1] if in1 else None
    want = oracle_taps[out_tap]
    got = ldm_model.run_block(name, x0, x1, poses=oracle_taps["poses"] if kind == "st" else None,
                              out_channels=want.shape[1], out_side=want.shape[2])
    e = rel_l2(got, want)
    log("ldm_module", module=name, kind=kind, rel_l2=e, max_rel=max_rel(got, want))
    assert e < BLOCK_TOL


def test_forward_vs_oracle(ldm_model, oracle_taps, golden):
    ref = torch.from_numpy(golden["ref_latent"])
    emb = ldm_model(ref.expand(N_HYP, -1, -1, -1), oracle_taps["poses"])
    e = rel_l2(emb, oracle_taps["emb"])
    log("ldm_forward_vs_oracle", emb_rel_l2=e, launches=ldm_model.last_launch_count)
    assert e < EMB_TOL_FP16


def test_taps_vs_oracle(ldm_model, oracle_taps, golden):
    """cumulative error along the network (informational thresholds: 2x the end-to-end tolerance)"""
    ref = torch.from_numpy(golden["ref_latent"])
    worst = 0.0
    for tap in ["input_blocks.0", "input_blocks.1.0", "input_blocks.1", "input_blocks.3", "input_blocks.5",
                "input_blocks.8", "middle_block", "output_blocks.2", "output_blocks.5", "output_blocks.8"]:
        got = ldm_model.debug_tap(ref, oracle_taps["poses"], tap)
        e = rel_l2(got, oracle_taps[tap])
        log("ldm_tap", tap=tap, rel_l2=e)
        worst = max(worst, e)
    assert worst < 2 * EMB_TOL_FP16


def test_sweep_golden(ldm_model, golden):
    """B=1, N=3 sweep with fused score / top-k against the unmodified reference's outputs."""
    ref = torch.from_numpy(golden["ref_latent"])
    qry = torch.from_numpy(golden["query_latent"])
    poses = torch.from_numpy(golden["all_relativeR"])
    out = ldm_model.sweep(ref, poses, qry, want_emb=True, k=3)
    e_emb = rel_l2(out["emb"][0], torch.from_numpy(golden["emb"]))
    e_sim = max_rel(out["sim"], torch.from_numpy(golden["similarity"]))
    order = torch.from_numpy(golden["similarity"]).argsort(dim=1, descending=True)
    log("ldm_sweep_golden", emb_rel_l2=e_emb, sim_max_rel=e_sim, topi=out["topi"].tolist(), ref_order=order.tolist())
    assert e_emb < EMB_TOL_FP16 and e_sim < SIM_TOL
    assert torch.equal(out["topi"].cpu(), order)
    # chunking / batching invariance: two references, chunk smaller than N
    ldm_model.set_chunk(2)
    try:
        out2 = ldm_model.sweep(torch.cat([ref, qry]), torch.cat([poses, poses]), torch.cat([qry, ref]), k=1)
    finally:
        ldm_model.set_chunk(8)
    assert torch.equal(out2["sim"][0], out["sim"][0])


def test_hoisted_prefix_is_bitwise_neutral(ldm_model, golden):
    """running the pose-independent prefix once per reference changes no bit of the result"""
    ref = torch.from_numpy(golden["ref_latent"])
    qry = torch.from_numpy(golden["query_latent"])
    poses = torch.from_numpy(golden["all_relativeR"])
    a = ldm_model.sweep(torch.cat([ref, qry]), torch.cat([poses, poses]), torch.cat([qry, ref]), want_emb=True, k=1)
    n_hoist = ldm_model.last_launch_count
    ldm_model.set_option("hoist", 0)
    try:
        b = ldm_model.sweep(torch.cat([ref, qry]), torch.cat([poses, poses]), torch.cat([qry, ref]), want_emb=True, k=1)
        n_plain = ldm_model.last_launch_count
    finally:
        ldm_model.set_option("hoist", 1)
    log("ldm_hoist", launches_hoisted=n_hoist, launches_plain=n_plain,
        max_abs_diff=float((a["emb"] - b["emb"]).abs().max()))
    assert torch.equal(a["emb"], b["emb"]) and torch.equal(a["sim"], b["sim"])


@pytest.fixture(scope="module")
def ldm_model_w2(ldm_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.ldm import UNetModelPose
    m = UNetModelPose(device="cuda:0", chunk=8, precision="fp16_w2")
    m.load_state_dict(ldm_sd)
    return m


def test_exact_weights_mode_meets_the_north_star_tolerance(ldm_model_w2, oracle_taps, golden):
    """precision="fp16_w2": embeddings within 1e-3 of the fp32 oracle AND of the unmodified reference's golden
    sweep, scores and ranking as in the fp16 mode"""
    ref = torch.from_numpy(golden["ref_latent"])
    emb = ldm_model_w2(ref.expand(N_HYP, -1, -1, -1), oracle_taps["poses"])
    e = rel_l2(emb, oracle_taps["emb"])
    qry = torch.from_numpy(golden["query_latent"])
    poses = torch.from_numpy(golden["all_relativeR"])
    out = ldm_model_w2.sweep(ref, poses, qry, want_emb=True, k=3)
    e_emb = rel_l2(out["emb"][0], torch.from_numpy(golden["emb"]))
    e_sim = max_rel(out["sim"], torch.from_numpy(golden["similarity"]))
    order = torch.from_numpy(golden["similarity"]).argsort(dim=1, descending=True)
    log("ldm_exact_weights", emb_rel_l2_vs_oracle=e, emb_rel_l2_vs_golden=e_emb, sim_max_rel=e_sim,
        launches=ldm_model_w2.last_launch_count)
    assert e < EMB_TOL and e_emb < EMB_TOL and e_sim < SIM_TOL
    assert torch.equal(out["topi"].cpu(), order)


def test_exact_weights_module_in_isolation(ldm_model_w2, oracle_taps):
    """a ResBlock (3x3 convs + folded identity / 1x1 skip K-segments) and a SpatialTransformer (q|k|v, GEGLU,
    residual linears) with the doubled segment list"""
    for name, kind, in0, in1, out_tap in [("input_blocks.4.0", "res", "input_blocks.3", None, "input_blocks.4.0"),
                                          ("input_blocks.4.1", "st", "input_blocks.4.0", None, "input_blocks.4"),
                                          ("output_blocks.2.0", "res", "output_blocks.1", "input_blocks.6", "output_blocks.2.0")]:
        want = oracle_taps[out_tap]
        got = ldm_model_w2.run_block(name, oracle_taps[in0], oracle_taps[in1] if in1 else None,
                                     poses=oracle_taps["poses"] if kind == "st" else None,
                                     out_channels=want.shape[1], out_side=want.shape[2])
        e = rel_l2(got, want)
        log("ldm_module_w2", module=name, rel_l2=e)
        assert e < BLOCK_TOL


def test_rejects_bad_input(ldm_model):
    from nope_b200 import _lib
    with pytest.raises(_lib.NopeError):
        ldm_model.run_block("no.such.module", torch.zeros(1, 256, 32, 32), out_channels=256, out_side=32)
    from nope_b200.ldm import UNetModelPose
    with pytest.raises(ValueError):
        UNetModelPose(channel_mult=(1, 2, 4, 8))
    # on an engine before finalize, where every option it has is accepted: names it does not have are errors,
    # the implementation switches included
    fresh = UNetModelPose(device="cuda:0", chunk=1)
    for name, value in (("fuse_geglu", 1), ("fold_residual", 1), ("wide_tiles", 1), ("conv_impl", 2),
                        ("attn_impl", 1)):
        with pytest.raises(_lib.NopeError):
            fresh.set_option(name, value)
    lib = _lib.load()
    for name in ("nope_ldm_set_impl", "nope_ldm_sweep"):
        assert not hasattr(lib, name), name


# ---------------------------------------------------------------- production batch sizes
# One module per (kind, resolution, one- or two-source) group that the network has, at a batch that gives the
# module's narrowest convolution (256-wide tiles) at least three tiles per CTA: the persistent kernel's
# second-and-later-tile paths.  At 8x8 two images share a tile and n = 197 leaves the last pair with a phantom peer.
# (module, kind, n, side of the GEMM, narrowest Cout, parities)
MANY_TILE_MODULES = [
    ("input_blocks.1.0", "res", 50, 32, 256, 1),            # identity skip
    ("input_blocks.5.0", "res", 100, 16, 512, 1),
    ("input_blocks.8.0", "res", 197, 8, 1024, 1),
    ("input_blocks.4.0", "res", 100, 16, 512, 1),           # 1x1 skip (the 32x32 one has two sources)
    ("input_blocks.7.0", "res", 197, 8, 1024, 1),
    ("output_blocks.8.0", "res", 50, 32, 256, 1),           # two sources, 1x1 skip
    ("output_blocks.3.0", "res", 100, 16, 512, 1),
    ("output_blocks.0.0", "res", 197, 8, 1024, 1),
    ("input_blocks.1.1", "st", 50, 32, 256, 1),
    ("input_blocks.4.1", "st", 100, 16, 512, 1),
    ("input_blocks.7.1", "st", 197, 8, 1024, 1),
    ("input_blocks.3.0.op", "resample", 200, 16, 256, 1),   # stride-2 3x3, 32 -> 16
    ("input_blocks.6.0.op", "resample", 397, 8, 512, 1),    # stride-2 3x3, 16 -> 8: odd m-tile count
    ("output_blocks.2.2.conv", "resample", 49, 8, 1024, 4), # folded nearest-x2 + 3x3, 8 -> 16: odd m-tile count
    ("output_blocks.5.2.conv", "resample", 25, 16, 512, 4), # folded nearest-x2 + 3x3, 16 -> 32
]
W2_MODULES = ("input_blocks.1.0", "input_blocks.4.0", "input_blocks.7.1")   # also run in precision="fp16_w2"
REF_SLICE = 8       # images per float64 oracle evaluation: its attention materialises [b, heads, tok, tok]


@pytest.fixture(scope="module")
def grid642(golden_dir):
    return torch.from_numpy(np.load(f"{golden_dir}/level2_642_b1.npz")["all_relativeR"])


def _oracle_module(sd, name, kind, x0, x1, poses):
    """the oracle's own module functions, on whatever dtype / device sd and the inputs have"""
    import torch.nn.functional as F
    from oracle import ldm_oracle
    if kind == "res":
        return ldm_oracle.res_block(x0 if x1 is None else torch.cat([x0, x1], 1), sd, name)
    if kind == "st":
        ctx = (poses @ sd["pose_mlp.0.weight"].t() + sd["pose_mlp.0.bias"])[:, None, :]
        return ldm_oracle.spatial_transformer(x0, ctx, sd, name)
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    if name.endswith(".op"):
        return F.conv2d(x0, w, b, stride=2, padding=1)
    return F.conv2d(F.interpolate(x0, scale_factor=2, mode="nearest"), w, b, padding=1)


def _like_tap(tap, n, gen):
    """seeded input with the per-channel mean and spread of an oracle tap"""
    m, s = tap.mean((0, 2, 3)), tap.std((0, 2, 3))
    return torch.randn((n,) + tuple(tap.shape[1:]), generator=gen) * s[:, None, None] + m[:, None, None]


@pytest.mark.parametrize("mod", MANY_TILE_MODULES, ids=lambda m: m[0])
def test_module_many_tiles(ldm_model, ldm_model_w2, ldm_sd, oracle_taps, grid642, mod):
    """run_block at production batch sizes against the oracle in float64 on the GPU: the worst per-image rel-L2,
    and slices of the batch (first, middle, last, odd start) equal the full run bit for bit"""
    from _util import min_many_tile_pairs, pair_tiles, rounds, worst_block_rel_l2
    name, kind, n, side, cout, n_par = mod
    pairs = pair_tiles(n, side, side, cout, 256, n_par)
    assert pairs >= min_many_tile_pairs(0), (name, n, pairs)
    spec = next(m for m in _modules() if m[0] == name)
    (in0, in1), out_tap = spec[2], spec[3]
    want = oracle_taps[out_tap]
    gen = torch.Generator().manual_seed(n + len(name))
    x0 = _like_tap(oracle_taps[in0], n, gen)
    x1 = _like_tap(oracle_taps[in1], n, gen) if in1 else None
    poses = grid642[0, :n] if kind == "st" else None
    dev = torch.device("cuda:0")
    d64 = lambda t: None if t is None else t.to(dev, torch.float64)
    sd = {k: d64(v) for k, v in ldm_sd.items() if k.startswith(name + ".") or k.startswith("pose_mlp.")}
    with torch.no_grad():
        ref = torch.cat([_oracle_module(sd, name, kind, d64(x0[i:i + REF_SLICE]),
                                        None if x1 is None else d64(x1[i:i + REF_SLICE]),
                                        None if poses is None else d64(poses[i:i + REF_SLICE]))
                         for i in range(0, n, REF_SLICE)])
    models = [("fp16", ldm_model)] + ([("fp16_w2", ldm_model_w2)] if name in W2_MODULES else [])
    for prec, m in models:
        run = lambda lo, hi: m.run_block(name, x0[lo:hi], None if x1 is None else x1[lo:hi],
                                         poses=None if poses is None else poses[lo:hi],
                                         out_channels=want.shape[1], out_side=ref.shape[2])
        got = run(0, n)
        e, img = worst_block_rel_l2(got, ref)
        log("ldm_module_many_tiles", module=name, precision=prec, n=n, pair_tiles=pairs, rounds=rounds(pairs, 0),
            worst_image_rel_l2=e,
            worst_image=img)
        assert e < BLOCK_TOL, (name, prec, "worst image", img, e)
        for lo, hi in [(0, REF_SLICE), (n // 3, 2 * n // 3), (n - 1, n), ((n // 2) | 1, n)]:
            part = run(lo, hi)
            assert torch.equal(part, got[lo:hi]), (name, prec, lo, hi)


SWEEP_HYPS = (0, 255, 256, 511, 512, 641)     # first / last of each 256-chunk of the 642 poses


@pytest.fixture(scope="module")
def ldm_model_256(ldm_sd):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.ldm import UNetModelPose
    return UNetModelPose(device="cuda:0", chunk=256).load_state_dict(ldm_sd)


def test_sweep_chunk256_bitwise_and_vs_oracle(ldm_model_256, ldm_sd, grid642):
    """The 642 poses of level2_642 at chunk 256 (chunks of 256 + 256 + 130), Q = 4 queries: (a) the same call twice,
    (b) chunks of 7 and 642 and (d) chosen hypotheses swept alone all give the same bits; those hypotheses are within
    EMB_TOL_FP16 / SIM_TOL of the oracle's forward in float64.  (c), four one-query sweeps equal to the Q = 4 sweep,
    is test_multi_query_gpu.test_ldm_multi_query_fused_scores_match_standalone on the same inputs."""
    from oracle import ldm_oracle
    from oracle import unet_oracle as orc
    m = ldm_model_256
    gen = torch.Generator().manual_seed(4)
    ref = torch.randn(1, 4, 32, 32, generator=gen)
    qry = torch.randn(1, 4, 4, 32, 32, generator=gen)
    poses = grid642
    base = m.sweep(ref, poses, qry, want_emb=True, k=5)
    keys = ("emb", "sim", "topv", "topi")

    def same(a, b, what):
        for k in keys:
            assert torch.equal(a[k], b[k]), (what, k)

    same(m.sweep(ref, poses, qry, want_emb=True, k=5), base, "second call")                  # (a)
    try:
        for chunk in (7, 642):                                                                 # (b)
            m.set_chunk(chunk)
            same(m.sweep(ref, poses, qry, want_emb=True, k=5), base, f"chunk {chunk}")
    finally:
        m.set_chunk(256)
    hyps = list(SWEEP_HYPS)
    for i in hyps:                                                                             # (d)
        alone = m.sweep(ref, poses[:, i:i + 1], qry, want_emb=True, k=1)
        assert torch.equal(alone["emb"][0, 0], base["emb"][0, i]), i
        assert torch.equal(alone["sim"][0, :, 0], base["sim"][0, :, i]), i
    dev = torch.device("cuda:0")
    sd = {k: v.to(dev, torch.float64) for k, v in ldm_sd.items()}
    with torch.no_grad():
        emb_o = ldm_oracle.ldm_forward(sd, ref.to(dev, torch.float64).expand(len(hyps), -1, -1, -1),
                                       poses[0, hyps].to(dev, torch.float64))
        sim_o = torch.stack([orc.l2_similarity(qry[:, q].to(dev, torch.float64), emb_o[None])[0]
                             for q in range(qry.shape[1])])                                  # [Q, hyps]
    e_emb = [rel_l2(base["emb"][0, i], emb_o[j]) for j, i in enumerate(hyps)]
    e_sim = max_rel(base["sim"][0][:, hyps], sim_o)
    log("ldm_sweep_chunk256", hyps=hyps, emb_rel_l2=e_emb, sim_max_rel=e_sim)
    assert max(e_emb) < EMB_TOL_FP16 and e_sim < SIM_TOL, (e_emb, e_sim)
