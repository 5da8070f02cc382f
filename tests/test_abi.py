"""CPU: the C-ABI library loads and exports every symbol include/dalm_b200.h declares (no compute without a GPU);
the ctypes table mirrors the header; product paths fail loudly without a GPU / library."""
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "dalm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dalm_b200_\w+)\s*\(", src)))


def test_library_builds_and_exports_header_symbols():
    import __graft_entry__ as g
    g.build()
    from dalm_b200 import _lib
    lib = _lib.load()
    names = _header_functions()
    assert len(names) >= 30
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r"\bT (dalm_b200_\w+)", out))
    for n in names:
        assert n in exported, f"{n} declared in the header but not exported"
        assert hasattr(lib, n)
    assert set(_lib.SIGNATURES) == set(names), set(_lib.SIGNATURES) ^ set(names)
    assert "sm_90a" in _lib.version()


def test_sass_is_hopper_native():
    """wgmma / TMA must really be in the binary (HGMMA / UTMALDG / UTMASTG), not a recompiled legacy path"""
    from dalm_b200 import _lib
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "UTMASTG"):
        assert mnemonic in sass, mnemonic


def test_no_cpu_fallback():
    from dalm_b200 import _lib, ops
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(_lib.DalmB200Error):
        ops.gemm(a, a)
    with pytest.raises(_lib.DalmB200Error):
        ops.inbatch_loss(torch.zeros(2, 4), torch.zeros(2, 4), 100.0)
    if not torch.cuda.is_available():
        from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E
        with pytest.raises(RuntimeError):
            AutoModelForRagE2E("x", "y")


def test_product_never_imports_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "dalm_b200")):
        for f in files:
            if f.endswith(".py") and re.search(r"^\s*(from|import)\s+oracle\b", open(os.path.join(dirpath, f)).read(), flags=re.M):
                bad.append(os.path.join(dirpath, f))
    assert not bad, bad
