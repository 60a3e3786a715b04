"""GPU: the per-launch profile of the two sweep engines (nope_unet_profile / nope_ldm_profile and their
*_profile_read), which bench.py's roofline reads.  Profiling must leave a sweep's outputs as they are, count only
the launches it times with their FLOPs, and start again from zero on every profile(True)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _sweep_inputs(seed, channels, B=1, N=5):
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(B, channels, 32, 32, generator=g) * 1.5
    poses = torch.randn(B, N, 6, generator=g)
    query = torch.randn(B, channels, 32, 32, generator=g) * 1.5
    return ref, poses, query


def _assert_same_outputs(a, b):
    for key in ("emb", "sim", "topv", "topi"):
        assert torch.equal(a[key], b[key]), key


def _profiled_sweep(model, ref, poses, query):
    """-> (profile_read() of one sweep with profiling on, the launch count of that sweep, profile_read() right after
    profile(True) again); the profiled sweep must return exactly what an unprofiled one does."""
    plain = model.sweep(ref, poses, query, want_emb=True, k=3)
    model.profile(True)
    timed = model.sweep(ref, poses, query, want_emb=True, k=3)
    prof, launches = model.profile_read(), model.last_launch_count
    _assert_same_outputs(plain, timed)
    model.profile(True)
    restarted = model.profile_read()
    model.profile(False)
    return prof, launches, restarted


def test_unet_profile():
    """conv_launches / conv_flops / conv_alg_flops of the UNet's convolutions: the split-precision mode executes
    more MMA work for the same algorithmic FLOPs.  At u_net_dim 64 the split-precision upsample convolutions take
    the epilogue of tiles up to 128 channels wide, so this also checks that their (hi, lo) outputs are reproducible."""
    from oracle import weights
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.unet import UNet
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sd = weights.make_unet_state_dict(seed=3, u_net_dim=64)
    ref, poses, query = _sweep_inputs(0, 8)
    reads = {}
    for precision in ("fp16", "parity"):
        unet = UNet(u_net_dim=64, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8),
                    pose_mlp_name="single_layer", device="cuda:0", precision=precision)
        unet.load_state_dict(sd)
        prof, launches, restarted = _profiled_sweep(unet, ref, poses, query)
        assert 0 < prof["conv_launches"] <= launches
        assert prof["conv_flops"] > 0 and prof["conv_alg_flops"] > 0
        assert restarted["conv_launches"] == 0 and restarted["conv_flops"] == 0 and restarted["conv_alg_flops"] == 0
        reads[precision] = prof
    assert reads["parity"]["conv_launches"] == reads["fp16"]["conv_launches"]
    assert reads["parity"]["conv_alg_flops"] == reads["fp16"]["conv_alg_flops"]
    assert reads["parity"]["conv_flops"] > reads["fp16"]["conv_flops"]


def test_ldm_profile():
    """launches / flops of the LDM's GEMM-shaped convolutions and its attention cores."""
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    m = UNetModelPose(device="cuda:0", chunk=8).load_state_dict(make_ldm_state_dict(seed=0))
    ref, poses, query = _sweep_inputs(1, 4)
    prof, launches, restarted = _profiled_sweep(m, ref, poses, query)
    gemm, attn = prof["gemm"], prof["attention"]
    assert gemm["launches"] > 0 and attn["launches"] > 0 and gemm["launches"] + attn["launches"] <= launches
    assert gemm["flops"] > 0 and attn["flops"] > 0
    for kind in ("gemm", "attention"):
        assert restarted[kind]["launches"] == 0 and restarted[kind]["flops"] == 0
