"""Host logic of native KvsAll training for TransE and RotatE on CPU: which norms B200TrainingJobKvsAll routes to the
fused CSR-label backward (under dropout), that the dot family's backward call is unchanged (no l_norm argument), and two training epochs
on an l_norm-aware stand-in of the engine against the reference job.  The CUDA path runs the same jobs in
tests/test_gpu_kvsall_distance.py."""
import contextlib

import pytest
import torch

from kge_b200 import hostenv

pytestmark = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")

import engine_stub  # noqa: E402
import jobs_util as ju  # noqa: E402

E, R, D = 53, 4, 16


@pytest.fixture(scope="module")
def splits():
    return ju.synthetic_splits(E, R, 150, 20, 20)


@contextlib.contextmanager
def _stub():
    """engine_stub.installed() with an l_norm-aware CSR-label backward; yields the keyword arguments of its calls."""
    from kge_b200 import engine

    calls = []

    def backward(model, combine, ent, rel, q, p, csr_offsets, csr_cols, loss="kl", offset=0.0, label_smoothing=0.0,
                 batch_size=None, **kw):
        calls.append(kw)
        e, r = ent.detach().clone().requires_grad_(True), rel.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            val = engine_stub.score_1vsN_loss_csr(model, combine, e, r, e, csr_offsets, csr_cols, q, p, loss, offset,
                                                  label_smoothing, kw.get("l_norm", 1.0))
            return torch.autograd.grad(val / (batch_size or q.numel()), (e, r))

    with engine_stub.installed():
        saved = engine.score_1vsN_loss_csr_backward
        engine.score_1vsN_loss_csr_backward = backward
        try:
            yield calls
        finally:
            engine.score_1vsN_loss_csr_backward = saved


def _job(model, splits, loss, eps, l_norm=None, job_class=None):
    extra = {"KvsAll.label_smoothing": eps}
    if l_norm is not None:
        extra[f"{model}.l_norm"] = l_norm
    torch.manual_seed(0)
    job = ju.make_job(model, E, R, D, splits, train_type="KvsAll", loss=loss, batch_size=16, forward_only=False,
                      extra=extra, job_class=job_class)
    return job


def _train(job, init):
    ju.copy_tables(init, job)
    losses = []
    for ep in range(2):
        job.epoch += 1
        if job.loader is None:
            job._prepare()
        ju.seed_all(10 + ep)
        losses.append(job.run_epoch()["avg_loss"])
    return losses


@pytest.mark.parametrize("model,l_norm,fused", [("transe", 1.0, True), ("transe", 2.0, True), ("rotate", 1.0, True),
                                               ("transe", 3.0, False), ("rotate", 2.0, False)])
def test_routing_by_norm(model, l_norm, fused, splits):
    """The CSR-label backward serves the covered norms under dropout; without dropout the distance family keeps the
    unmodified step (stored dense scores, native dense backward), which is the faster one there."""
    init = _job(model, splits, "kl", 0.1, l_norm)
    with _stub() as calls:
        job = _job("b200_" + model, splits, "kl", 0.1, l_norm, job_class="B200TrainingJobKvsAll")
        assert job.model.b200_kvsall_native_backward_ok(dropout=True) == fused
        assert not job.model.b200_kvsall_native_backward_ok()
        _train(job, init)
    assert not calls


def test_dot_family_backward_call_is_unchanged(splits):
    init = _job("distmult", splits, "kl", 0.1)
    with _stub() as calls:
        _train(_job("b200_distmult", splits, "kl", 0.1, job_class="B200TrainingJobKvsAll"), init)
    assert calls and all("l_norm" not in kw for kw in calls)


@pytest.mark.parametrize("model,l_norm,loss,eps", [("transe", 1.0, "kl", 0.1), ("transe", 2.0, "bce", 0.0),
                                                   ("rotate", 1.0, "bce", 0.1)])
def test_two_epochs_track_the_reference(model, l_norm, loss, eps, splits):
    init = _job(model, splits, loss, eps, l_norm)
    ref = _train(_job(model, splits, loss, eps, l_norm), init)
    with _stub() as calls:
        job = _job("b200_" + model, splits, loss, eps, l_norm, job_class="B200TrainingJobKvsAll")
        job.model.b200_kvsall_native_backward_ok = lambda dropout=False: True      # the route taken under dropout
        got = _train(job, init)
    assert calls and all(kw.get("l_norm") == l_norm for kw in calls)
    assert got == pytest.approx(ref, rel=1e-5)
    assert ref[1] < ref[0]
