"""CPU: the lifecycle the five weight-holding engines share, without a device -- every *_create fails with an error
message (no fallback), and _lib.build_engine destroys an engine whose build fails part way."""
import ctypes as C

import pytest
import torch

from nope_b200 import _lib

CREATE = {"unet": (192, 8, 32, 0), "encoder": (8, 0), "vae": (0,), "vae_decoder": (0,), "ldm": (256, 512, 4, 32, 0)}


@pytest.mark.parametrize("kind", sorted(CREATE))
def test_create_without_a_gpu_is_an_error(kind):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    create = getattr(lib, f"nope_{kind}_create")
    assert create(None, *CREATE[kind]) != 0
    assert lib.nope_last_error() == b"check failed: out != nullptr -- null out pointer"
    h = C.c_void_p()
    assert create(C.byref(h), *CREATE[kind]) != 0
    assert h.value is None
    msg = lib.nope_last_error()
    assert len(msg) > 0 and b"null out pointer" not in msg, msg


class _FakeLib:
    """the engine entry points build_engine calls, with load_tensor failing on the key `bad`"""

    def __init__(self, bad):
        self.bad, self.calls = bad, []

    def __getattr__(self, name):
        def fn(h, *args):
            self.calls.append(name)
            if name.endswith("_create"):
                h._obj.value = 1234
            return 1 if name.endswith("_load_tensor") and args[0] == self.bad else 0
        return fn

    def nope_last_error(self):
        return b"refused"


@pytest.mark.parametrize("bad", [b"b", None])
def test_build_engine_destroys_the_engine_when_a_step_fails(monkeypatch, bad):
    fake = _FakeLib(bad)
    monkeypatch.setattr(_lib, "load", lambda: fake)
    configured = []
    tensors = [("a", torch.zeros(2, 3, dtype=torch.float64)), ("b", torch.ones(4)), ("c", torch.ones(()))]
    if bad is None:
        h = _lib.build_engine("vae", (0,), tensors, lambda lib, h: configured.append(h.value))
        assert h.value == 1234
        assert fake.calls == ["nope_vae_create"] + ["nope_vae_load_tensor"] * 3 + ["nope_vae_finalize"]
    else:
        with pytest.raises(_lib.NopeError, match="refused"):
            _lib.build_engine("vae", (0,), tensors, lambda lib, h: configured.append(h.value))
        assert fake.calls == ["nope_vae_create"] + ["nope_vae_load_tensor"] * 2 + ["nope_vae_destroy"]
    assert configured == [1234]
