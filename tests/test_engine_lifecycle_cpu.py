"""CPU: the lifecycle the five weight-holding engines share, without a device -- every *_create fails with an error
message (no fallback), _lib.build_engine destroys an engine whose build fails part way, and _lib.Engine, the handle
owner of the Python classes, makes, rebuilds and destroys its one handle in order."""
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


# ------------------------------------------------------------------ _lib.Engine, the handle owner of the Python classes
@pytest.fixture
def fake(monkeypatch):
    lib = _FakeLib(None)
    monkeypatch.setattr(_lib, "load", lambda: lib)
    return lib


def _configure(lib, h):
    lib.calls.append(f"configure {h.value}")


TENSORS = [("a", torch.zeros(2)), ("b", torch.ones(3))]
BUILD = ["nope_ldm_create", "configure 1234"] + ["nope_ldm_load_tensor"] * 2 + ["nope_ldm_finalize"]


def test_engine_makes_one_weightless_configured_handle(fake):
    e = _lib.Engine("ldm")
    h = e.handle((256, 0), _configure)
    assert e.handle((256, 0), _configure) is h and h.value == 1234 and not e.finalized
    assert fake.calls == ["nope_ldm_create", "configure 1234"]            # configured, nothing loaded
    e.destroy()


def test_engine_rebuild_destroys_the_old_handle_first(fake):
    e = _lib.Engine("ldm")
    e.handle((0,), _configure)
    e.build((0,), TENSORS, _configure)
    assert e.finalized
    e.build((0,), TENSORS, _configure)
    assert fake.calls == ["nope_ldm_create", "configure 1234"] + ["nope_ldm_destroy"] + BUILD + \
        ["nope_ldm_destroy"] + BUILD
    e.destroy()


def test_engine_failed_build_leaves_no_handle(fake):
    e = _lib.Engine("ldm")
    fake.bad = b"b"
    with pytest.raises(_lib.NopeError, match="refused"):
        e.build((0,), TENSORS, _configure)
    assert e.h is None and not e.finalized
    assert fake.calls == BUILD[:-1] + ["nope_ldm_destroy"]        # the load of `b` fails
    fake.bad, fake.calls = None, []
    assert e.build((0,), TENSORS, _configure).value == 1234 and e.finalized
    assert fake.calls == BUILD
    e.destroy()


def test_engine_second_destroy_is_a_no_op(fake):
    e = _lib.Engine("vae")
    e.build((0,), TENSORS)
    e.destroy()
    e.destroy()
    assert e.h is None and not e.finalized
    assert fake.calls.count("nope_vae_destroy") == 1 and fake.calls[-1] == "nope_vae_destroy"


def test_engine_del_does_not_raise_when_load_fails(fake, monkeypatch):
    e = _lib.Engine("vae")
    e.build((0,), TENSORS)

    def fail():
        raise _lib.NopeError("no library")
    monkeypatch.setattr(_lib, "load", fail)
    e.__del__()
    assert e.h is None
    del e
