"""CPU: the C-ABI library loads and exports every symbol include/b200sv.h declares; the ctypes table covers them all.
No compute call is made (no GPU here)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200sv.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sv_[a-z0-9_]+)\s*\(", text)))


def test_header_is_plain_c(tmp_path):
    import subprocess
    src = tmp_path / "t.c"
    src.write_text('#include "b200sv.h"\nint main(void){ b200sv_logsv_params p = {0}; (void)p; return B200SV_VERSION == 0; }\n')
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", f"-I{ROOT}/include", str(src)], check=True)


def test_library_exports_every_declared_symbol():
    from stochvolmodels_b200 import _capi
    if not os.path.exists(_capi.LIB_PATH):
        from stochvolmodels_b200._build import build_library
        build_library()
    lib = ctypes.CDLL(_capi.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b200sv.h but not exported"
    bound = set(_capi.SIGNATURES) | set(_capi._MISC)
    assert set(declared) == bound, (set(declared) ^ bound)
    loaded = _capi.load_library()
    assert loaded.b200sv_version() == 100
    assert loaded.b200sv_last_error() is not None


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from stochvolmodels_b200 import _capi
    monkeypatch.setattr(_capi, "_lib", None)
    monkeypatch.setattr(_capi, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _capi.load_library()


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under stochvolmodels_b200/ may reference it."""
    pkg = os.path.join(ROOT, "stochvolmodels_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), os.path.join(dirpath, f)


def test_library_calls_stay_in_their_abi_modules():
    """engine.py marshals the host-level entry points and multi_gpu.py the device-level ones; no other product module calls the library
    or builds raw pointers."""
    pkg = os.path.join(ROOT, "stochvolmodels_b200")
    allowed = {os.path.join(pkg, f) for f in ("engine.py", "multi_gpu.py", "_capi.py")}
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith(".py") and path not in allowed:
                text = open(path).read()
                for pattern in ("C.call(", "_capi.call(", ".ctypes.data_as("):
                    assert pattern not in text, f"{pattern} in {path}"
