"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/monoport_b200.h declares
(no compute calls -- there is no GPU here)."""
import os
import re

from conftest import ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "monoport_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mp_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from monoport_b200 import build, _lib
    path = build.build()
    assert os.path.exists(path)
    lib = _lib.load()
    syms = _header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), "library does not export %s" % s
    assert sorted(_lib.SIGNATURES) == syms, "ctypes table and header disagree"
    assert lib.mp_version() >= 100


def test_built_for_sm90a_only():
    import subprocess
    from monoport_b200 import _lib
    out = subprocess.run(["cuobjdump", "--list-elf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from monoport_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    import pytest
    with pytest.raises(_lib.MonoportLibraryError):
        _lib.load()


def test_cpu_tensors_are_rejected_not_silently_computed():
    """No CPU fallback: eval-mode query on CPU tensors must raise."""
    import pytest
    import torch
    from monoport_b200.modeling import PIFuNetG
    net = PIFuNetG().eval()
    with pytest.raises(RuntimeError):
        net.query([[torch.zeros(1, 256, 8, 8)]], torch.zeros(1, 3, 4), calibs=torch.eye(4)[None])
    from monoport_b200.recon import forward_vertices, marching_cubes
    with pytest.raises(RuntimeError):
        forward_vertices(torch.zeros(1, 1, 9, 9, 9))
    with pytest.raises(RuntimeError):
        marching_cubes(torch.zeros(9, 9, 9))
