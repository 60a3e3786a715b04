"""CPU: the C-ABI library loads and exports every symbol include/nope_b200.h declares."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "nope_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nope_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_loads():
    from nope_b200 import build
    build.build()
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_abi_version() == _lib.EXPECTED_ABI == 2
    assert lib.nope_build_arch() == b"sm_90a"


def test_exports_match_header():
    from nope_b200 import _lib
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/nope_b200.h but not exported"
    assert set(names) == set(_lib.SIGNATURES), set(names) ^ set(_lib.SIGNATURES)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from nope_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.NopeError):
        _lib.load()


def test_no_gpu_means_error_not_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import ctypes as C
    from nope_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.nope_unet_create(C.byref(h), 192, 8, 32, 0) != 0
    assert len(lib.nope_last_error()) > 0


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "nope_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
