"""CPU: libesr_b200.so builds for sm_90a, loads, and exports every symbol include/esr_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "esr_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(esr_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from esr_b200 import build, _lib
    path = build.build()
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), f"{n} declared in esr_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in esr_b200/_lib.py"
    assert lib.esr_version() >= 100


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from esr_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    import pytest
    with pytest.raises(_lib.ESRError):
        _lib.lib()
