"""CPU tests of argument validation in b200kge_sample_uniform_filtered and b200kge_filter_index_build: each call passes
one bad argument and must be refused with B200KGE_ERR_INVALID before anything reaches a device.  Every buffer is host
memory, so an argument that slipped past validation would surface as a CUDA error code instead."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="host buffers only: runs where there is no GPU")

INVALID = -1
N, K, V, NK = 4, 3, 10, 2
BAD = ("vocab", "slot", "n", "K", "num_keys", "out", "triples", "keys", "offsets", "values")


@pytest.fixture(scope="module")
def lib():
    from kge_b200.build import build_native
    from kge_b200 import _lib

    build_native()
    return _lib.load()


def _call(lib, bad=None):
    keep = [np.zeros(N * 3, np.int64), np.array([0, 1, 0, 2], np.int64), np.array([0, 1, 2], np.int64),
            np.array([3, 4], np.int64), np.zeros(N * K, np.int64)]
    tri, keys, offs, vals, out = (a.ctypes.data for a in keep)
    a = dict(vocab=V, slot=2, n=N, K=K, num_keys=NK, out=out, triples=tri, keys=keys, offsets=offs, values=vals)
    if bad is not None:
        a[bad] = {"vocab": 0, "slot": 3, "n": -1, "K": -1, "num_keys": -1}.get(bad)
    rc = lib.b200kge_sample_uniform_filtered(1, 2, a["vocab"], a["n"], a["K"], a["triples"], a["slot"], a["keys"],
                                             a["offsets"], a["values"], a["num_keys"], a["out"], None)
    del keep
    return rc


def test_valid_arguments_pass_validation(lib):
    assert _call(lib) != INVALID, lib.b200kge_last_error()


@pytest.mark.parametrize("bad", BAD)
def test_bad_argument_is_refused(lib, bad):
    assert _call(lib, bad) == INVALID, lib.b200kge_last_error()


@pytest.mark.parametrize("offsets", [[0, 3, -1], [0, -2, 1], [2, 1, 5]])
def test_decreasing_offsets_are_refused_before_values_are_read(lib, offsets):
    """values is NULL: a builder that read values before checking every offset would fault instead of refusing."""
    import ctypes as C

    keys = np.array([0, 1, 0, 2], np.int64)
    offs = np.array(offsets, np.int64)
    out = np.zeros(8, np.int64)
    nk, mx = C.c_int64(0), C.c_int64(0)
    rc = lib.b200kge_filter_index_build(keys.ctypes.data, offs.ctypes.data, None, 2, V, out.ctypes.data,
                                        out.ctypes.data, out.ctypes.data, C.byref(nk), C.byref(mx))
    assert rc == INVALID and b"decrease" in lib.b200kge_last_error()
