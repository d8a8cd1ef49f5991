"""CPU tests of argument validation in the C entry points that take whole tables: each call passes one bad argument
and must be refused with B200KGE_ERR_INVALID before anything reaches a device.  Every buffer is host memory, so an
argument that slipped past validation would surface as a CUDA error code instead."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="host buffers only: runs where there is no GPU")

INVALID = -1
COMPLEX, TRANSE = 0, 5
BCE = 1
E, R, D, N, K = 10, 3, 8, 4, 2


@pytest.fixture(scope="module")
def lib():
    from kge_b200.build import build_native
    from kge_b200 import _lib

    build_native()
    return _lib.load()


class Args:
    """A valid call's arguments (host buffers) with at most one of them made bad."""

    def __init__(self, bad=None):
        from kge_b200 import _lib

        self.model, self.l_norm, self.loss, self.num_rel, self.mask_dir = COMPLEX, 1.0, BCE, R, None
        dim, ld, rel_rows, p_ent = D, D, 2 * R, 0.1
        idx = None
        if bad == "model":
            self.model = 99
        elif bad == "odd_dim":
            dim = D - 1
        elif bad == "l_norm":
            self.model, self.l_norm = TRANSE, 0.0
        elif bad == "loss":
            self.loss = 42
        elif bad == "dropout":
            p_ent = 1.0
        elif bad == "rel_rows":
            rel_rows = R
        elif bad == "num_rel":
            self.num_rel = -R
        elif bad == "mask_dir":
            self.mask_dir = 2
        self._keep = []
        self.ent_buf = self._f32(E, ld)
        self.rel_buf = self._f32(2 * R, ld)
        if bad == "idx":
            idx = self._i64(E).ctypes.data
        ent = _lib.Rows(self.ent_buf.ctypes.data, idx, E, ld, dim)
        rel = _lib.Rows(self.rel_buf.ctypes.data, None, rel_rows, ld, dim)
        self._keep += [ent, rel]
        self.ent = None if bad == "null" else C.byref(ent)
        self.rel = C.byref(rel)
        self.lde = D - 2 if bad == "lde" else ld
        self.ldr = ld
        drop = _lib.Dropout(p_ent, 0.1, 1234, 0, 0)
        self._keep.append(drop)
        self.drop = C.byref(drop)
        self.triples = self._i64(N * 3).ctypes.data
        self.idx = self._i64(N).ctypes.data
        self.neg = self._i64(N * K).ctypes.data
        self.csr_off = self._i64(N + 1).ctypes.data
        self.csr_col = self._i64(N).ctypes.data
        self.f = self._f32(N, E).ctypes.data          # scores / grad_scores / loss / rank outputs
        self.grad = None if bad == "no_grad" else self.f      # a dropout backward without grad_scores
        self.d_ent = self._f32(E, ld).ctypes.data
        self.d_rel = self._f32(2 * R, ld).ctypes.data
        self.ws = self._f32(1 << 16)
        self.wsp, self.wsn = self.ws.ctypes.data, self.ws.nbytes

    def _f32(self, *shape):
        a = np.zeros(shape, dtype=np.float32)
        self._keep.append(a)
        return a

    def _i64(self, n):
        a = np.zeros(n, dtype=np.int64)
        self._keep.append(a)
        return a


def _grad(a):
    return (a.d_ent, a.lde, a.d_rel, a.ldr, a.wsp, a.wsn, None)


# entry point (":mode" for the training entries that take several) -> (call, the bad arguments it must refuse).  Modes:
# plain, dropout, reciprocal relations (num_relations > 0) and both for the 1vsAll step; plain and dropout with mask_dir
# = combine (sp_) or not for the CSR backward; the in-kernel BCE gradient, a given gradient and dropout for NS.
COMMON = ("null", "idx", "model", "odd_dim")


def _fwd_1vsall(reciprocal, drop):
    return lambda L, a: L.b200kge_train_1vsall_forward(a.model, a.l_norm, 0, a.ent, a.rel, a.num_rel if reciprocal else 0,
                                                       a.triples, N, a.loss, 0.0, a.drop if drop else None, a.f, a.wsp,
                                                       a.wsn, None)


def _bwd_1vsall(reciprocal, drop):
    return lambda L, a: L.b200kge_train_1vsall_backward(a.model, a.l_norm, a.ent, a.rel, a.num_rel if reciprocal else 0,
                                                        a.triples, N, a.loss, 0.0, a.drop if drop else None, *_grad(a))


def _csr_bwd(mask_dir, drop):
    return lambda L, a: L.b200kge_score_1vsN_loss_csr_backward(a.model, 0, a.mask_dir if a.mask_dir is not None else
                                                               mask_dir, a.l_norm, a.ent, a.rel, a.idx, a.idx, N,
                                                               a.csr_off, a.csr_col, 0.0, a.loss, 0.0, N,
                                                               a.drop if drop else None, *_grad(a))


def _ns_bwd(drop, grad):
    return lambda L, a: L.b200kge_ns_backward(a.model, a.l_norm, a.ent, a.rel, a.triples, 0, a.neg, N, K, 0,
                                              a.drop if drop else None, a.grad if grad else None, E, 0.0, N, *_grad(a))


ENTRIES = {
    "train_1vsall_forward:plain": (_fwd_1vsall(False, False), COMMON + ("l_norm", "loss")),
    "train_1vsall_backward:plain": (_bwd_1vsall(False, False), COMMON + ("l_norm", "loss", "lde")),
    "train_1vsall_forward:dropout": (_fwd_1vsall(False, True), COMMON + ("l_norm", "loss", "dropout")),
    "train_1vsall_backward:dropout": (_bwd_1vsall(False, True), COMMON + ("l_norm", "loss", "lde", "dropout")),
    "train_1vsall_forward:reciprocal": (_fwd_1vsall(True, False),
                                        COMMON + ("l_norm", "loss", "rel_rows", "num_rel")),
    "train_1vsall_forward:reciprocal+dropout": (_fwd_1vsall(True, True),
                                                COMMON + ("l_norm", "loss", "rel_rows", "num_rel", "dropout")),
    "train_1vsall_backward:reciprocal": (_bwd_1vsall(True, False),
                                         COMMON + ("l_norm", "loss", "lde", "rel_rows", "num_rel")),
    "train_1vsall_backward:reciprocal+dropout": (_bwd_1vsall(True, True),
                                                 COMMON + ("l_norm", "loss", "lde", "rel_rows", "num_rel", "dropout")),
    "score_1vsN_backward": (
        lambda L, a: L.b200kge_score_1vsN_backward(a.model, 0, a.l_norm, a.ent, a.rel, a.idx, a.idx, N, a.f, E,
                                                   *_grad(a)),
        COMMON + ("l_norm", "lde")),
    "score_1vsN_loss_csr_backward:plain": (_csr_bwd(1, False), COMMON + ("loss", "lde")),
    "score_1vsN_loss_csr_dropout:mask_dir=sp_": (
        lambda L, a: L.b200kge_score_1vsN_loss_csr_dropout(a.model, 0, 0, a.l_norm, 0, a.ent, a.rel, a.idx, a.idx, N,
                                                           a.csr_off, a.csr_col, N, 0.0, a.loss, 0.0, a.drop, a.f,
                                                           None, a.wsp, a.wsn, None),
        COMMON + ("dropout",)),
    "score_1vsN_loss_csr_dropout:mask_dir=_po": (
        lambda L, a: L.b200kge_score_1vsN_loss_csr_dropout(a.model, 0, 1, a.l_norm, 0, a.ent, a.rel, a.idx, a.idx, N,
                                                           a.csr_off, a.csr_col, N, 0.0, a.loss, 0.0, a.drop, a.f,
                                                           None, a.wsp, a.wsn, None),
        COMMON + ("dropout",)),
    "score_1vsN_loss_csr_backward:dropout,mask_dir=sp_": (_csr_bwd(0, True), COMMON + ("loss", "lde", "dropout", "mask_dir")),
    "score_1vsN_loss_csr_backward:dropout,mask_dir=_po": (_csr_bwd(1, True),
                                                 COMMON + ("loss", "lde", "dropout", "mask_dir")),
    "ns_backward:bce": (_ns_bwd(False, False), COMMON + ("l_norm", "lde")),
    "ns_backward:grad_scores": (_ns_bwd(False, True), COMMON + ("l_norm", "lde")),
    "ns_score_dropout": (
        lambda L, a: L.b200kge_ns_score_dropout(a.model, a.l_norm, a.ent, a.rel, a.triples, 0, a.neg, N, K, 0, a.drop,
                                                a.f, E, None),
        COMMON + ("l_norm", "dropout")),
    "ns_backward:dropout": (_ns_bwd(True, True), COMMON + ("l_norm", "lde", "dropout", "no_grad")),
    "rank_sp_po_eval": (
        lambda L, a: L.b200kge_rank_sp_po_eval(a.model, a.l_norm, 0, a.ent, a.rel, a.num_rel, a.idx, a.idx, a.idx, N,
                                               a.f, a.idx, a.csr_off, a.csr_col, None, None, 0.0, 0.0, a.d_ent,
                                               a.d_rel, a.f, a.wsp, a.wsn, None),
        COMMON + ("l_norm", "rel_rows")),
}


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_valid_arguments_pass_validation(lib, entry):
    """The unmodified arguments get past validation (without a device they then fail further on)."""
    call, _ = ENTRIES[entry]
    a = Args()
    assert call(lib, a) != INVALID, lib.b200kge_last_error()


@pytest.mark.parametrize("entry,bad", [(e, b) for e in sorted(ENTRIES) for b in ENTRIES[e][1]])
def test_bad_argument_is_refused(lib, entry, bad):
    call, _ = ENTRIES[entry]
    a = Args(bad)
    assert call(lib, a) == INVALID, lib.b200kge_last_error()


@pytest.mark.parametrize("entry", ["score_1vsN_loss", "loss_dense", "score_1vsN_loss_csr"])
def test_bad_loss_kind_is_refused(lib, entry):
    from kge_b200 import _lib

    a = Args()
    q = _lib.Rows(a.ent_buf.ctypes.data, None, N, D, D)
    cand = _lib.Rows(a.ent_buf.ctypes.data, None, E, D, D)
    labels = _lib.Labels(a.idx, None, 0)
    if entry == "score_1vsN_loss":
        rc = lib.b200kge_score_1vsN_loss(COMPLEX, 0, 1.0, 0, C.byref(q), C.byref(q), C.byref(cand), N,
                                         C.byref(labels), 42, 0.0, a.f, None, a.wsp, a.wsn, None)
    elif entry == "loss_dense":
        rc = lib.b200kge_loss_dense(a.f, E, N, E, C.byref(labels), 42, 0.0, a.f, None, a.wsp, a.wsn, None)
    else:
        rc = lib.b200kge_score_1vsN_loss_csr(COMPLEX, 0, 1.0, 0, C.byref(q), C.byref(q), C.byref(cand), N, a.csr_off,
                                             a.csr_col, N, 0.0, 42, 0.0, a.f, None, a.wsp, a.wsn, None)
    assert rc == INVALID, lib.b200kge_last_error()
