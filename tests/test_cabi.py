"""CPU tests of the boundary: the C-ABI library builds for sm_90a, loads, exports every symbol
include/b200kge.h declares, and refuses to compute without a GPU (no CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from kge_b200.build import build_native
    from kge_b200 import _lib

    build_native()
    return _lib.load()


def test_header_symbols_all_exported(lib):
    from kge_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "b200kge.h")).read()
    declared = set(re.findall(r"\b(b200kge_[a-z0-9_A-Z]+)\s*\(", hdr))
    assert declared, "no declarations found"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.b200kge_version() == 101


def test_sass_is_hopper_native():
    import shutil
    import subprocess

    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    from kge_b200._lib import LIB_PATH

    sass = subprocess.run(["cuobjdump", "-sass", LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG"):   # wgmma / TMA
        assert mnemonic in sass, mnemonic


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback(lib):
    from kge_b200 import KgeModel, engine

    assert lib.b200kge_device_ok() != 0
    assert b"no CPU fallback" in lib.b200kge_last_error() or b"not sm_90" in lib.b200kge_last_error()
    m = KgeModel("complex", 10, 2, 8)
    idx = torch.tensor([0, 1])
    with pytest.raises(RuntimeError):
        m.score_sp(idx, idx)
    with pytest.raises(RuntimeError):
        engine.loss_dense(torch.zeros(2, 3), idx)


def test_workspace_bytes_monotone(lib):
    a = lib.b200kge_workspace_bytes(0, 128, 1000, 128, 0)
    b = lib.b200kge_workspace_bytes(0, 1024, 14541, 512, 0)
    c = lib.b200kge_workspace_bytes(0, 1024, 14541, 512, 1)
    assert 0 < a < b < c
