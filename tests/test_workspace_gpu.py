"""GPU: the workspace growth the UNet, LDM and template encoder engines share (grow_workspace, csrc/engine.cuh).

Pinned here: an engine that grows its workspace for a larger call and then serves a smaller one computes, at every
step, exactly what a fresh engine computes for that call alone; and a growth whose allocation fails raises NopeError
and leaves an engine whose next call grows again and matches a fresh engine bit for bit."""
import pytest
import torch

from nope_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SMALL, LARGE = (1, 3, 1), (2, 7, 2)          # (references B, poses N, queries Q) of one sweep


@pytest.fixture(scope="module")
def unet_state():
    from nope_b200.synth_weights import make_unet_state_dict
    return make_unet_state_dict(seed=0)


@pytest.fixture(scope="module")
def ldm_state():
    from nope_b200.synth_weights import make_ldm_state_dict
    return make_ldm_state_dict(seed=0)


def _unet(state, chunk=4, precision="fp16"):
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.unet import UNet
    u = UNet(u_net_dim=192, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8), device=DEV,
             chunk=chunk, precision=precision)
    u.load_state_dict(state)
    return u


def _sweep_inputs(shape, channels, seed=3):
    B, N, Q = shape
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(B, channels, 32, 32, generator=g)
    poses = torch.randn(B, N, 6, generator=g)
    qry = torch.randn(B, Q, channels, 32, 32, generator=g)
    return ref.to(DEV), poses.to(DEV), qry.to(DEV)


def _unet_own_workspace(u, shape, k=2):
    """nope_unet_sweep_multi without UNet.reserve: the engine sizes a workspace of its own"""
    ref, poses, qry = _sweep_inputs(shape, 8)
    B, N, Q = shape
    out = {"emb": torch.empty((B, N, 8, 32, 32), device=DEV), "sim": torch.empty((B, Q, N), device=DEV),
           "topv": torch.empty((B, Q, k), device=DEV), "topi": torch.empty((B, Q, k), device=DEV, dtype=torch.int64)}
    with torch.cuda.device(DEV):
        _lib.check(_lib.load().nope_unet_sweep_multi(
            u._handle(), _lib.ptr(ref), _lib.ptr(poses), B, N, _lib.ptr(qry), Q, _lib.ptr(out["emb"]),
            _lib.ptr(out["sim"]), k, _lib.ptr(out["topv"]), _lib.ptr(out["topi"]), 0, _lib.stream(DEV)))
    return out


def _python_sweep(m, shape, channels, k=2):
    """the Python owner's sweep (UNet.sweep sizes a caller-owned workspace through UNet.reserve)"""
    return m.sweep(*_sweep_inputs(shape, channels), want_emb=True, k=k)


def _equal(a, b):
    return all(torch.equal(a[n], b[n]) for n in ("emb", "sim", "topv", "topi"))


def _regrowth(make, run):
    """small -> large -> small on one engine, each result equal to a fresh engine's"""
    grown = make()
    fresh = {SMALL: run(make(), SMALL), LARGE: run(make(), LARGE)}
    for shape in (SMALL, LARGE, SMALL):
        assert _equal(run(grown, shape), fresh[shape]), shape


@pytest.mark.parametrize("owner", ["engine", "caller"])
def test_unet_regrowth_equals_fresh_engines(unet_state, owner):
    run = _unet_own_workspace if owner == "engine" else (lambda u, shape: _python_sweep(u, shape, 8))
    _regrowth(lambda: _unet(unet_state), run)


def test_ldm_regrowth_equals_fresh_engines(ldm_state):
    from nope_b200.ldm import UNetModelPose
    _regrowth(lambda: UNetModelPose(device=DEV, chunk=4).load_state_dict(ldm_state),
              lambda m, shape: _python_sweep(m, shape, 4))


def test_encoder_regrowth_equals_fresh_engines():
    from nope_b200.encoder import FeatureExtractor
    torch.manual_seed(0)
    weights = FeatureExtractor(descriptor_size=8).state_dict()

    def encoder():
        fe = FeatureExtractor(descriptor_size=8)
        fe.load_state_dict(weights)
        return fe.to(DEV)

    g = torch.Generator().manual_seed(4)
    images = {n: (torch.rand(n, 3, 256, 256, generator=g) * 2 - 1).to(DEV) for n in (2, 5)}
    fresh = {n: encoder().encode_image(images[n]) for n in (2, 5)}
    grown = encoder()
    for n in (2, 5, 2):
        assert torch.equal(grown.encode_image(images[n]), fresh[n]), n


def test_unet_failed_growth_leaves_a_working_engine(unet_state):
    """A workspace larger than the device cannot be allocated: the sweep raises NopeError, and the engine's next
    sweep grows a workspace again instead of running on the freed one"""
    chunk = 4096
    u = _unet(unet_state, chunk=chunk, precision="parity")
    lib, h = _lib.load(), u._handle()
    total = torch.cuda.get_device_properties(DEV).total_memory
    one, two = lib.nope_unet_workspace_bytes(h, chunk, 1, 0), lib.nope_unet_workspace_bytes(h, chunk, 2, 0)
    B = (total - one) // (two - one) + 2
    assert lib.nope_unet_workspace_bytes(h, chunk, B, 0) > total
    before = _unet_own_workspace(u, SMALL)          # the engine holds a workspace when the growth fails
    ref = torch.zeros((B, 8, 32, 32), device=DEV)   # correctly sized inputs of B references, one pose each
    poses = torch.zeros((B, 1, 6), device=DEV)
    with torch.cuda.device(DEV), pytest.raises(_lib.NopeError, match="workspace"):
        _lib.check(lib.nope_unet_sweep_multi(h, _lib.ptr(ref), _lib.ptr(poses), B, 1, None, 1, None, None, 0, None,
                                             None, 0, _lib.stream(DEV)))
    del ref, poses
    after = _unet_own_workspace(u, SMALL)
    fresh = _unet_own_workspace(_unet(unet_state, chunk=chunk, precision="parity"), SMALL)
    assert _equal(after, fresh) and _equal(before, fresh)
