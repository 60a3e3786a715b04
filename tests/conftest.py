import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (H100); run with -m gpu")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def seeded_state_dict():
    """Full reference-schema state_dict (UNet + encoder) from the seeded recipe."""
    from oracle import weights
    return weights.make_full_state_dict(seed=0)


@pytest.fixture(scope="session")
def gpu_model_parity(seeded_state_dict):
    """The same model in the split-precision mode (exact weights + hi/lo activations): the mode that
    carries the north-star 1e-3 embedding tolerance."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.model import build_model
    m = build_model(device="cuda:0", precision="parity")
    m.load_state_dict(seeded_state_dict)
    return m.eval()


@pytest.fixture(scope="session")
def gpu_model(seeded_state_dict):
    """nope_b200 PoseConditional on cuda:0 with the seeded weights (session-wide)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nope_b200.model import build_model
    m = build_model(device="cuda:0")
    m.load_state_dict(seeded_state_dict)
    impl = os.environ.get("NOPE_CONV_IMPL", "tcgen05_2cta")   # "simt": bring-up twin on CUDA cores
    m.u_net.set_conv_impl(impl)
    return m.eval()
