"""KvsAll's s_o query type (relation prediction) on CPU: which models and options B200TrainingJobKvsAll serves natively,
two training epochs of the plugin job with sp_ + s_o + _po against the unmodified reference job on oracle-backed
stand-ins of engine.score_so_loss_csr / score_so_loss_csr_backward (tests/so_oracle.py), the argument refusals of the two
C entry points and their workspace sizes.  The CUDA path runs the same jobs in tests/test_gpu_kvsall_so.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from kge_b200 import hostenv

import so_oracle as so  # noqa: E402

needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")

E, R, D = 53, 6, 16
P_ENT, P_REL = 0.4, 0.2
REL = 1e-5
QTYPES = {"KvsAll.query_types.sp_": True, "KvsAll.query_types.s_o": True, "KvsAll.query_types._po": True}


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 150, 20, 20)


@pytest.fixture()
def stub():
    with so.installed() as calls:
        calls["so"] = calls["so_dropout"] = 0
        yield calls


def _job(model, splits, loss, extra=None, job_class=None, dropout=False, imports=()):
    import jobs_util as ju

    cfg = dict(QTYPES)
    if dropout:
        cfg.update({f"{model}.entity_embedder.dropout": P_ENT, f"{model}.relation_embedder.dropout": P_REL})
    cfg.update(extra or {})
    return ju.make_job(model, E, R, D, splits, train_type="KvsAll", loss=loss, batch_size=32, forward_only=False,
                       extra=cfg, job_class=job_class, imports=imports)


def _train(job, init, subbatch=None):
    import jobs_util as ju

    ju.copy_tables(init, job)
    if subbatch:
        job._max_subbatch_size = subbatch
    losses = []
    for ep in range(2):
        job.epoch += 1
        if job.loader is None:
            job._prepare()
        ju.seed_all(10 + ep)
        losses.append(job.run_epoch()["avg_loss"])
    return losses


def _pair(model, splits, loss, extra=None, dropout=False, subbatch=None):
    import jobs_util as ju

    torch.manual_seed(0)
    init = ju.make_job(model, E, R, D, splits, train_type="KvsAll", loss=loss, batch_size=32, extra=QTYPES)
    ref = _job(model, splits, loss, extra, dropout=dropout)
    if dropout:
        so.patch_reference_job(ref, P_ENT, P_REL)
    plugin = _job("b200_" + model, splits, loss, extra, "B200TrainingJobKvsAll", dropout)
    return _train(ref, init, subbatch), _train(plugin, init, subbatch), plugin


@needs_ref
@pytest.mark.parametrize("model,loss,extra,dropout,subbatch", [
    ("complex", "kl", None, False, None),
    ("complex", "bce", {"train.loss_arg": 0.5}, False, None),
    ("complex", "kl", {"KvsAll.label_smoothing": 0.1}, False, None),
    ("complex", "kl", None, True, None),
    ("complex", "bce", {"KvsAll.label_smoothing": 0.1}, True, 7),
    ("distmult", "kl", None, False, 5),
    ("simple", "bce", None, True, None),
    ("cp", "kl", None, True, None),
    ("rescal", "kl", {"KvsAll.label_smoothing": 0.1}, False, None),
], ids=lambda v: str(v))
def test_two_epochs_match_the_reference_job(model, loss, extra, dropout, subbatch, splits, stub):
    """sp_ + s_o + _po: the s_o rows take the new entries (never smoothed), the losses match the unmodified job."""
    ref, plugin, job = _pair(model, splits, loss, extra, dropout, subbatch)
    assert stub["so"] > 0 and stub["so_dropout"] == (stub["so"] if dropout else 0)
    assert plugin == pytest.approx(ref, rel=REL)


@needs_ref
def test_forward_only_takes_the_fused_forward(splits, stub):
    import jobs_util as ju

    job = _job("b200_complex", splits, "kl", job_class="B200TrainingJobKvsAll")
    job.is_forward_only = True
    ju.run_forward_epoch(job)
    assert stub["so"] > 0


@needs_ref
@pytest.mark.parametrize("model,extra,imports", [
    ("b200_transe", None, ()),
    ("b200_rotate", None, ()),
    ("b200_transe", None, ()),
    ("b200_complex", {"b200_complex.precision": "tf32"}, ()),
    ("reciprocal_relations_model", {"reciprocal_relations_model.base_model.type": "b200_complex"}, ("b200_complex",)),
], ids=["transe", "rotate", "transe-dropout", "complex-tf32", "reciprocal"])
def test_uncovered_settings_make_no_s_o_call(model, extra, imports, splits, stub, request):
    """TransE, RotatE (no s_o fold), a precision outside auto / fp32 / f16x3 and the reciprocal wrapper (whose reference
    raises for s_o) keep today's route: no call of the new entries."""
    drop = "dropout" in request.node.callspec.id
    job = _job(model, splits, "kl", extra, "B200TrainingJobKvsAll", dropout=drop, imports=imports)
    try:
        job.epoch += 1
        job._prepare()
        job.run_epoch()
    except Exception:                  # the reciprocal wrapper's reference step raises for s_o
        assert model == "reciprocal_relations_model"
    assert stub["so"] == 0


@needs_ref
def test_predicate(splits, stub):
    job = _job("b200_complex", splits, "kl", job_class="B200TrainingJobKvsAll")
    assert job.model.b200_kvsall_so_ok()
    job.model.b200_backward = "reference"
    assert not job.model.b200_kvsall_so_ok()


# ---- the C entry points: argument refusals and workspace sizes (host buffers, no device) ------------------------------
INVALID, UNSUPPORTED = -1, -2
COMPLEX, DISTMULT, CP, RESCAL, TRANSE, ROTATE = 0, 1, 3, 4, 5, 6
N = 4
cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="host buffers only: runs where there is no GPU")


@pytest.fixture(scope="module")
def lib():
    from kge_b200.build import build_native
    from kge_b200 import _lib

    build_native()
    return _lib.load()


class SoArgs:
    """A valid s_o call's arguments (host buffers) with at most one of them made bad."""

    def __init__(self, bad=None):
        from kge_b200 import _lib

        self.model, self.loss, self.batch = COMPLEX, 1, N
        dim, rdim, ld = D, D, D
        idx = None
        p_ent = 0.1
        self._keep = []
        if bad == "model":
            self.model = 99
        elif bad == "odd_dim":
            dim = D - 1
        elif bad == "rel_dim":
            rdim = D // 2
        elif bad == "loss":
            self.loss = 42
        elif bad == "dropout":
            p_ent = 1.0
        elif bad == "batch_size":
            self.batch = 0
        elif bad == "transe":
            self.model = TRANSE
        elif bad == "rotate":
            self.model, rdim = ROTATE, D // 2
        self.ent_buf, self.rel_buf = self._f32(E, ld), self._f32(R, ld)
        if bad == "idx":
            idx = self._i64(E).ctypes.data
        ent = _lib.Rows(self.ent_buf.ctypes.data, idx, E, ld, dim)
        rel = _lib.Rows(self.rel_buf.ctypes.data, None, R, ld, rdim)
        self._keep += [ent, rel]
        self.ent = None if bad == "null" else C.byref(ent)
        self.rel = C.byref(rel)
        self.lde = D - 2 if bad == "lde" else ld
        drop = _lib.Dropout(p_ent, 0.1, 1234, 0, 0)
        self._keep.append(drop)
        self.drop = C.byref(drop)
        self.idx = self._i64(N).ctypes.data
        self.csr_off = self._i64(N + 1).ctypes.data
        self.csr_col = self._i64(N).ctypes.data
        self.f = self._f32(N, E).ctypes.data
        self.d_ent, self.d_rel = self._f32(E, ld).ctypes.data, self._f32(R, ld).ctypes.data
        self.ws = self._f32(1 << 16)

    def _f32(self, *shape):
        a = np.zeros(shape, dtype=np.float32)
        self._keep.append(a)
        return a

    def _i64(self, n):
        a = np.zeros(n, dtype=np.int64)
        self._keep.append(a)
        return a


def _fwd(drop):
    return lambda L, a: L.b200kge_score_so_loss_csr(a.model, 1.0, 0, a.ent, a.rel, a.idx, a.idx, N, a.csr_off, a.csr_col,
                                                    N, a.loss, 0.0, a.drop if drop else None, a.f, None,
                                                    a.ws.ctypes.data, a.ws.nbytes, None)


def _bwd(drop):
    return lambda L, a: L.b200kge_score_so_loss_csr_backward(a.model, 1.0, a.ent, a.rel, a.idx, a.idx, N, a.csr_off,
                                                             a.csr_col, a.loss, 0.0, a.batch, a.drop if drop else None,
                                                             a.d_ent, a.lde, a.d_rel, D, a.ws.ctypes.data, a.ws.nbytes,
                                                             None)


COMMON = ("null", "idx", "model", "odd_dim", "rel_dim", "loss")
ENTRIES = {
    "score_so_loss_csr:plain": (_fwd(False), COMMON),
    "score_so_loss_csr:dropout": (_fwd(True), COMMON + ("dropout",)),
    "score_so_loss_csr_backward:plain": (_bwd(False), COMMON + ("lde", "batch_size")),
    "score_so_loss_csr_backward:dropout": (_bwd(True), COMMON + ("lde", "batch_size", "dropout")),
}


@cpu_only
@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_valid_arguments_pass_validation(lib, entry):
    a = SoArgs()
    assert ENTRIES[entry][0](lib, a) not in (INVALID, UNSUPPORTED), lib.b200kge_last_error()


@cpu_only
@pytest.mark.parametrize("entry,bad", [(e, b) for e in sorted(ENTRIES) for b in ENTRIES[e][1]])
def test_bad_argument_is_refused(lib, entry, bad):
    a = SoArgs(bad)
    assert ENTRIES[entry][0](lib, a) == INVALID, lib.b200kge_last_error()


@cpu_only
@pytest.mark.parametrize("entry", sorted(ENTRIES))
@pytest.mark.parametrize("model", ["transe", "rotate"])
def test_distance_family_is_unsupported(lib, entry, model):
    """TransE and RotatE have no s_o fold: refused before any launch (host buffers would fail any launch)."""
    a = SoArgs(model)
    assert ENTRIES[entry][0](lib, a) == UNSUPPORTED, lib.b200kge_last_error()


# (model, n, R, D, nnz): every workspace the two entries take on these shapes, with and without dropout
SHAPES = [(m, n, r, d, nnz) for m in (COMPLEX, DISTMULT, 2, CP, RESCAL)
          for n, r, d, nnz in ((0, 5, 16, 0), (7, 5, 16, 9), (600, 237, 128, 1500), (1024, 237, 512, 2500))]


def _k(model, d):
    return d * d if model == RESCAL else (d // 2 if model == CP else d)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "m{}-n{}-R{}-D{}-nnz{}".format(*s))
def test_workspace_bytes(lib, shape):
    """The size covers the folded queries and the larger of the forward's loss steps and the backward block; with
    dropout also the masked copies and their gradients; it grows with n and nnz."""
    model, n, r, d, nnz = shape
    k = _k(model, d)
    ldq = (k + 31) // 32 * 32
    plain = lib.b200kge_score_so_loss_csr_workspace_bytes(model, n, r, d, nnz, 0)
    drop = lib.b200kge_score_so_loss_csr_workspace_bytes(model, n, r, d, nnz, 1)
    assert plain >= 2 * n * ldq * 4 + lib.b200kge_workspace_bytes(DISTMULT, n, r, k, 0) // 2
    assert drop - plain == 2 * (2 * n * d * 4 + r * k * 4 + 3 * 256)
    assert lib.b200kge_score_so_loss_csr_workspace_bytes(model, n + 1, r, d, nnz, 0) > plain
    assert lib.b200kge_score_so_loss_csr_workspace_bytes(model, n, r, d, nnz + 100, 0) >= plain
