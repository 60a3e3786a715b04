"""GPU: the lifecycle the five weight-holding engines share (csrc/engine.cuh, _lib.build_engine) -- the state_dict
checks of *_load_tensor with errors that name the engine and the key, the missing-key check of *_finalize, no loads
after finalize -- and the Python owners: a reload rebuilds the engine, a failed build leaves no engine behind."""
import ctypes as C

import pytest
import torch

from nope_b200 import _lib

pytestmark = pytest.mark.gpu

NAMES = {"unet": "UNet", "encoder": "encoder", "vae": "VAE", "vae_decoder": "VAE decoder", "ldm": "LDM"}
CREATE = {"unet": (192, 8, 32, 0), "encoder": (8, 0), "vae": (0,), "vae_decoder": (0,), "ldm": (256, 512, 4, 32, 0)}


def _schema(kind):
    from nope_b200 import synth_weights as W
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.vae import vae_decoder_param_shapes, vae_param_shapes
    if kind == "unet":
        return dict(W.unet_param_shapes(192, 8, 6))
    if kind == "encoder":
        return {k: tuple(v.shape) for k, v in FeatureExtractor(descriptor_size=8).state_dict().items()
                if not (k.endswith("num_batches_tracked") or k.startswith("backbone.fc."))}
    if kind == "vae":
        return dict(vae_param_shapes())
    if kind == "vae_decoder":
        return dict(vae_decoder_param_shapes())
    return dict(W.ldm_param_shapes())


def _create(kind):
    h = C.c_void_p()
    _lib.check(getattr(_lib.load(), f"nope_{kind}_create")(C.byref(h), *CREATE[kind]))
    return h


def _load(kind, h, key, shape):
    t = torch.zeros(shape, dtype=torch.float32)
    dims = (C.c_int64 * t.dim())(*t.shape)
    lib = _lib.load()
    rc = getattr(lib, f"nope_{kind}_load_tensor")(h, key.encode(), C.c_void_p(t.data_ptr()), dims, t.dim())
    return rc, lib.nope_last_error().decode()


def _refused(kind, rc, msg, *needles):
    assert rc != 0 and msg.startswith(NAMES[kind] + ": "), msg
    for n in needles:
        assert n in msg, msg


@pytest.mark.parametrize("kind", sorted(NAMES))
def test_load_tensor_checks_name_the_engine_and_the_key(kind):
    schema = _schema(kind)
    key = sorted(schema)[0]
    shape = tuple(schema[key])
    lib = _lib.load()
    h = _create(kind)
    try:
        _refused(kind, *_load(kind, h, "no.such.key", (1,)), "unexpected", "'no.such.key'")
        _refused(kind, *_load(kind, h, key, shape + (1,)), "rank mismatch", f"'{key}'")
        _refused(kind, *_load(kind, h, key, (shape[0] + 1,) + shape[1:]), "shape mismatch", f"'{key}'")
        assert _load(kind, h, key, shape)[0] == 0
        rc = getattr(lib, f"nope_{kind}_finalize")(h)
        msg = lib.nope_last_error().decode()
        _refused(kind, rc, msg, "state_dict is missing '")
        assert msg.split("'")[1] in schema and msg.split("'")[1] != key
    finally:
        getattr(lib, f"nope_{kind}_destroy")(h)


@pytest.fixture(scope="module")
def finalized():
    """one finalized engine of every kind, built through the Python owners"""
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict, make_unet_state_dict, make_vae_state_dict
    from nope_b200.unet import UNet
    from nope_b200.vae import VAE_StableDiffusion
    dev = torch.device("cuda:0")
    unet = UNet(u_net_dim=192, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8), device=dev)
    unet.load_state_dict(make_unet_state_dict(seed=0))
    fe = FeatureExtractor(descriptor_size=8).to(dev)
    vae = VAE_StableDiffusion(device=dev).load_state_dict(make_vae_state_dict(seed=0, decoder=True))
    ldm = UNetModelPose(device=dev, chunk=4).load_state_dict(make_ldm_state_dict(seed=0))
    owners = (unet, fe, vae, ldm)        # the handles below live as long as these
    yield owners, {"unet": unet._handle(), "encoder": fe._engine(dev), "vae": vae._engine(),
                   "vae_decoder": vae._decoder(), "ldm": ldm._handle()}


@pytest.mark.parametrize("kind", sorted(NAMES))
def test_no_load_after_finalize(finalized, kind):
    schema = _schema(kind)
    key = sorted(schema)[0]
    h = finalized[1][kind]
    _refused(kind, *_load(kind, h, key, tuple(schema[key])), "already finalized", f"'{key}'")
    lib = _lib.load()
    _refused(kind, getattr(lib, f"nope_{kind}_finalize")(h), lib.nope_last_error().decode(), "already finalized")


def _sweep_inputs(C_lat, seed=5):
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(2, C_lat, 32, 32, generator=g)
    qry = torch.randn(2, C_lat, 32, 32, generator=g)
    poses = torch.randn(2, 3, 6, generator=g)
    return ref, poses, qry


def _same_sweep(a, b, C_lat):
    ref, poses, qry = _sweep_inputs(C_lat)
    x = a.sweep(ref, poses, qry, want_emb=True, k=2)
    y = b.sweep(ref, poses, qry, want_emb=True, k=2)
    return all(torch.equal(x[n], y[n]) for n in ("emb", "sim", "topv", "topi"))


def test_unet_reload_equals_a_fresh_load():
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.synth_weights import make_unet_state_dict
    from nope_b200.unet import UNet

    def unet():
        return UNet(u_net_dim=192, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8),
                    device="cuda:0", chunk=4)
    twice = unet()
    twice.load_state_dict(make_unet_state_dict(seed=0))
    twice.load_state_dict(make_unet_state_dict(seed=1))
    once = unet()
    once.load_state_dict(make_unet_state_dict(seed=1))
    assert _same_sweep(twice, once, 8)


def test_ldm_reload_equals_a_fresh_load():
    from nope_b200.ldm import UNetModelPose
    from nope_b200.synth_weights import make_ldm_state_dict
    twice = UNetModelPose(device="cuda:0", chunk=4, precision="fp16_w2")
    twice.load_state_dict(make_ldm_state_dict(seed=0))
    twice.load_state_dict(make_ldm_state_dict(seed=1))
    once = UNetModelPose(device="cuda:0", chunk=4, precision="fp16_w2")
    once.load_state_dict(make_ldm_state_dict(seed=1))
    assert _same_sweep(twice, once, 4)


def test_failed_encoder_build_leaves_no_engine(monkeypatch):
    from nope_b200.encoder import FeatureExtractor
    lib = _lib.load()
    destroyed, destroy = [], lib.nope_encoder_destroy
    monkeypatch.setattr(lib, "nope_encoder_destroy", lambda h: (destroyed.append(h.value), destroy(h))[1])
    fe = FeatureExtractor(descriptor_size=8).to("cuda:0")
    x = torch.rand(2, 3, 256, 256, device="cuda:0") * 2 - 1
    w = fe.projector[3].weight
    good = w.data
    w.data = torch.zeros(8, 255, 1, 1, device="cuda:0")
    with pytest.raises(_lib.NopeError, match="encoder: .*'projector.3.weight'"):
        fe.encode_image(x)
    assert fe._h is None and len(destroyed) == 1 and destroyed[0] is not None
    w.data = good
    out = fe.encode_image(x)
    assert fe._h is not None and out.shape == (2, 8, 32, 32) and torch.isfinite(out).all()
