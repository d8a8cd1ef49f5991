"""Embedding dropout of the 1vsAll / KvsAll job plugins on CPU: properties of the mask mirror (tests/dropout_oracle.py)
and the plugin's routing, with kge_b200.engine replaced by oracle-backed stand-ins that apply the mirror's masks.  The
reference jobs draw the same masks through dropout modules patched in by this test only.  The CUDA kernels are checked
against the same mirror in tests/test_gpu_dropout.py."""
import math

import pytest
import torch

import dropout_oracle as dro
from kge_b200 import hostenv

E, R, D = 53, 4, 16
P_ENT, P_REL = 0.3, 0.1
# fp32 summation order (the reference's cdist for TransE, sub-batch rescaling); a wrong mask moves the loss by O(1)
REL = 1e-4


# ---- the mirror ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.3, 0.5, 0.9])
def test_keep_rate(p):
    m = dro.mask(p, seed=1234, call=7, stream=2, rows=96, dim=37)
    n = m.numel()
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(m.float().mean().item() - (1 - p)) < 5 * sigma


def test_masks_are_keyed_by_stream_call_and_row():
    base = dro.mask(0.5, 99, 3, 0, 8, 12)
    assert not torch.equal(base, dro.mask(0.5, 99, 3, 1, 8, 12))           # stream
    assert not torch.equal(base, dro.mask(0.5, 99, 4, 0, 8, 12))           # call
    assert not torch.equal(base, dro.mask(0.5, 98, 3, 0, 8, 12))           # seed
    assert not torch.equal(base[:4], base[4:])                              # rows
    # the global row keys the element: a window at row_base 3 sees the same rows as the full draw
    assert torch.equal(dro.mask(0.5, 99, 3, 0, 5, 12, row_base=3), base[3:])
    # p = 0 keeps everything
    assert bool(dro.mask(0.0, 99, 3, 0, 8, 12).all())


def test_apply_scales_kept_values():
    x = torch.randn(6, 10)
    y = dro.apply(x, 0.3, 5, 6, 4, row_base=2)
    m = dro.mask(0.3, 5, 6, 4, 6, 10, row_base=2)
    assert torch.equal(y[~m], torch.zeros_like(y[~m]))
    assert torch.equal(y[m], x[m] * torch.tensor(1.0 / 0.7, dtype=torch.float32))


# ---- plugin routing --------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 150, 20, 20)


@pytest.fixture()
def stub():
    with dro.installed():
        dro.calls["dropout"] = 0
        yield


def _job(model, splits, train_type, loss, p_ent=P_ENT, p_rel=P_REL, job_class=None, batch_size=32, extra=None):
    import jobs_util as ju

    cfg = {f"{model}.entity_embedder.dropout": p_ent, f"{model}.relation_embedder.dropout": p_rel}
    cfg.update(extra or {})
    return ju.make_job(model, E, R, D, splits, train_type=train_type, loss=loss, batch_size=batch_size,
                       forward_only=False, extra=cfg, job_class=job_class)


def _train_pair(model, splits, train_type, loss, job_class, subbatch=None, extra=None):
    """Two training epochs of the reference job (mirror masks patched in) and of the plugin job from the same tables."""
    import jobs_util as ju

    torch.manual_seed(0)
    init = ju.make_job(model, E, R, D, splits, train_type=train_type, loss=loss, batch_size=32, extra=extra)
    out = {}
    for tag in ("ref", "plugin"):
        if tag == "ref":
            job = dro.patch_reference_job(_job(model, splits, train_type, loss, extra=extra), P_ENT, P_REL)
        else:
            job = _job("b200_" + model, splits, train_type, loss, job_class=job_class, extra=extra)
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
        out[tag] = losses
    return out


@needs_ref
@pytest.mark.parametrize("subbatch", [None, 10])
@pytest.mark.parametrize("model,loss", [("complex", "kl"), ("transe", "bce")])
def test_1vsall_job_with_dropout(model, loss, subbatch, splits, stub):
    out = _train_pair(model, splits, "1vsAll", loss, "B200TrainingJob1vsAll", subbatch)
    assert dro.calls["dropout"] > 0                       # the dropout entry points ran
    assert out["plugin"] == pytest.approx(out["ref"], rel=REL)


@needs_ref
@pytest.mark.parametrize("subbatch", [None, 5])
@pytest.mark.parametrize("loss,eps", [("kl", 0.0), ("bce", 0.1)])
def test_kvsall_job_with_dropout(loss, eps, subbatch, splits, stub):
    out = _train_pair("distmult", splits, "KvsAll", loss, "B200TrainingJobKvsAll", subbatch,
                      extra={"KvsAll.label_smoothing": eps})
    assert dro.calls["dropout"] > 0
    assert out["plugin"] == pytest.approx(out["ref"], rel=REL)


@needs_ref
def test_backward_uses_the_forward_key(splits, stub):
    from kge_b200 import engine

    seen = []
    fwd, bwd = engine.train_1vsall_forward, engine.train_1vsall_backward

    def f(*a, dropout=None, **kw):
        seen.append(("f", dropout))
        return fwd(*a, dropout=dropout, **kw)

    def b(*a, dropout=None, **kw):
        seen.append(("b", dropout))
        return bwd(*a, dropout=dropout, **kw)

    engine.train_1vsall_forward, engine.train_1vsall_backward = f, b
    job = _job("b200_complex", splits, "1vsAll", "kl", job_class="B200TrainingJob1vsAll")
    job.epoch += 1
    job._prepare()
    job.run_epoch()
    assert len(seen) == 2 * len(job.loader)
    for (kf, key_f), (kb, key_b) in zip(seen[::2], seen[1::2]):
        assert (kf, kb) == ("f", "b") and key_f is not None and key_f == key_b
    calls = [k.call for _, k in seen[::2]]
    assert len(set(calls)) == len(calls)                   # a fresh key per sub-batch
    assert seen[0][1].seed == torch.initial_seed() and seen[0][1][:2] == pytest.approx((P_ENT, P_REL))


@needs_ref
def test_negative_sampling_job_with_dropout_keeps_the_reference_step(splits, stub):
    job = _job("b200_complex", splits, "negative_sampling", "kl", job_class="B200TrainingJobNegativeSampling",
               extra={"negative_sampling.num_samples.s": 3, "negative_sampling.num_samples.o": 3})

    def refuse(*a, **kw):
        raise AssertionError("the fused NS step must not run with dropout")

    job.model.loss_negatives = job.model.score_negatives = refuse
    job.epoch += 1
    job._prepare()
    assert math.isfinite(job.run_epoch()["avg_loss"])
    assert dro.calls["dropout"] == 0


@needs_ref
@pytest.mark.parametrize("train_type,job_class", [("1vsAll", "B200TrainingJob1vsAll"),
                                                  ("KvsAll", "B200TrainingJobKvsAll")])
def test_dropout_zero_and_eval_mode_keep_the_existing_routes(train_type, job_class, splits, stub):
    from kge_b200.plugin.jobs import _fused_model

    job = _job("b200_distmult", splits, train_type, "kl", p_ent=0.0, p_rel=0.0, job_class=job_class)
    job.epoch += 1
    job._prepare()
    job.run_epoch()
    assert dro.calls["dropout"] == 0
    assert job.model.b200_dropout_rates() is None

    job = _job("b200_distmult", splits, train_type, "kl", job_class=job_class)
    job.model.train()
    assert job.model.b200_dropout_rates() == pytest.approx((P_ENT, P_REL)) and _fused_model(job.model) is None
    job.model.eval()
    assert job.model.b200_dropout_rates() is None and _fused_model(job.model) is job.model
    import jobs_util as ju

    ju.run_valid(job)                                       # EntityRankingJob: eval mode
    assert dro.calls["dropout"] == 0
