"""Reciprocal-relations training through the job plugins on CPU: routing (p + R, o as the second half's query, labels
s, the _po mask streams), the fall-throughs, and two-epoch parity with the unmodified wrapper job.  kge_b200.engine is
replaced by oracle-backed stand-ins (tests/engine_stub.py, tests/dropout_oracle.py and the reciprocal ones below); the
CUDA kernels are checked against fp64 in tests/test_gpu_reciprocal.py."""
import pytest
import torch

import dropout_oracle as dro
import ns_dropout_oracle as nsd
from kge_b200 import hostenv

E, R, D = 53, 4, 16
P_ENT, P_REL = 0.3, 0.1
REL = 1e-4

pytestmark = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")

calls = []


def _recip_loss(model, ent, rel, tri, num_rel, loss, offset, key, l_norm):
    from oracle import kge_oracle as orc

    tri = tri.long()
    s, p, o = tri[:, 0], tri[:, 1], tri[:, 2]
    total = 0.0
    for direction, a, pr, lab in ((0, s, p, o), (1, o, p + num_rel, s)):
        q, r, t = ent[a], rel[pr], ent
        if key is not None:
            sq, sr, st = dro.DIR_STREAMS[direction]
            q = dro.apply(q, key.p_ent, key.seed, key.call, sq, key.row_base)
            r = dro.apply(r, key.p_rel, key.seed, key.call, sr, key.row_base)
            t = dro.apply(t, key.p_ent, key.seed, key.call, st, 0)
        x = orc.score_emb(model, q, r, t, "sp_", l_norm)
        total = total + (orc.bce_loss(x, lab, offset) if loss == "bce" else orc.kl_loss(x, lab))
    return total / tri.shape[0]


def _recip_forward(model, ent, rel, triples, num_relations, loss="bce", offset=0.0, l_norm=1.0, precision="auto",
                   dropout=None):
    assert rel.shape[0] == 2 * num_relations
    calls.append(("1vsall", int(num_relations), dropout is not None))
    return _recip_loss(model, ent, rel, triples, num_relations, loss, offset, dropout, l_norm)


def _recip_backward(model, ent, rel, triples, num_relations, loss="bce", offset=0.0, l_norm=1.0, dropout=None):
    return dro.grads(lambda e, r: _recip_loss(model, e, r, triples, num_relations, loss, offset, dropout, l_norm),
                     ent, rel)[1:]


def _kvs_loss(model, combine, streams, ent, rel, q, p, offs, cols, loss, offset, eps, key, l_norm=1.0):
    from oracle import kge_oracle as orc

    sq, sr, st = dro.DIR_STREAMS[0 if streams == "sp_" else 1]
    a = dro.apply(ent[q.long()], key.p_ent, key.seed, key.call, sq, key.row_base)
    r = dro.apply(rel[p.long()], key.p_rel, key.seed, key.call, sr, key.row_base)
    t = dro.apply(ent, key.p_ent, key.seed, key.call, st, 0)
    x = orc.score_emb(model, a, r, t, "sp_", l_norm) if combine == "sp_" else orc.score_emb(model, t, r, a, "_po", l_norm)
    y = torch.zeros(x.shape, dtype=x.dtype)
    rows = torch.repeat_interleave(torch.arange(x.shape[0]), offs[1:] - offs[:-1])
    y.index_put_((rows, cols.long()), torch.ones(len(rows), dtype=x.dtype), accumulate=True)
    if eps > 0:
        y = orc.kvsall_smooth_labels(y, eps)
    return orc.bce_loss(x, y, offset) if loss == "bce" else orc.kl_loss(x, y)


def _wrap_csr(fwd, bwd):
    def csr(model, combine, q_tab, rel, cand_tab, offs, cols, q=None, p=None, loss="kl", offset=0.0, label_smoothing=0.0,
            l_norm=1.0, precision="auto", return_rows=False, dropout=None, dropout_streams=None):
        calls.append(("kvsall", combine, q.clone(), p.clone(), dropout_streams))
        if dropout is None or dropout_streams is None:
            kw = {} if dropout is None else {"dropout": dropout}
            return fwd(model, combine, q_tab, rel, cand_tab, offs, cols, q, p, loss, offset, label_smoothing, l_norm,
                       precision, return_rows, **kw)
        return _kvs_loss(model, combine, dropout_streams, cand_tab, rel, q, p, offs, cols, loss, offset,
                         label_smoothing, dropout, l_norm)

    def csr_backward(model, combine, ent, rel, q, p, offs, cols, loss="kl", offset=0.0, label_smoothing=0.0,
                     batch_size=None, dropout=None, dropout_streams=None):
        if dropout is None or dropout_streams is None:
            kw = {} if dropout is None else {"dropout": dropout}
            return bwd(model, combine, ent, rel, q, p, offs, cols, loss, offset, label_smoothing, batch_size, **kw)
        bs = batch_size or q.numel()
        return dro.grads(lambda e, r: _kvs_loss(model, combine, dropout_streams, e, r, q, p, offs, cols, loss, offset,
                                                label_smoothing, dropout) / bs, ent, rel)[1:]
    return csr, csr_backward


@pytest.fixture()
def stub(monkeypatch):
    with nsd.installed():
        from kge_b200 import engine

        monkeypatch.setattr(engine, "train_1vsall_reciprocal_forward", _recip_forward)
        monkeypatch.setattr(engine, "train_1vsall_reciprocal_backward", _recip_backward)
        fwd, bwd = _wrap_csr(engine.score_1vsN_loss_csr, engine.score_1vsN_loss_csr_backward)
        monkeypatch.setattr(engine, "score_1vsN_loss_csr", fwd)
        monkeypatch.setattr(engine, "score_1vsN_loss_csr_backward", bwd)
        calls.clear()
        yield


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 150, 20, 20)


def _make(bm, train_type, loss, splits, job_class=None, extra=None, dropout=False):
    import jobs_util as ju

    cfg = {"reciprocal_relations_model.base_model.type": bm}
    if dropout:
        cfg.update({f"{bm}.entity_embedder.dropout": P_ENT, f"{bm}.relation_embedder.dropout": P_REL})
    cfg.update(extra or {})
    return ju.make_job("reciprocal_relations_model", E, R, D, splits, train_type=train_type, loss=loss, batch_size=32,
                       forward_only=False, imports=(bm,), extra=cfg, job_class=job_class)


def _pair(base, train_type, loss, job_class, splits, extra=None, dropout=False, subbatch=None):
    import jobs_util as ju

    torch.manual_seed(0)
    init = _make(base, train_type, loss, splits, extra=extra)
    out = {}
    for tag, bm, cls in (("ref", base, None), ("plugin", "b200_" + base, job_class)):
        job = _make(bm, train_type, loss, splits, cls, extra, dropout)
        if tag == "ref" and dropout:
            dro.patch_reference_job(job, P_ENT, P_REL)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a)
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


@pytest.mark.parametrize("subbatch", [None, 10])
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("base,loss", [("complex", "kl"), ("transe", "bce"), ("cp", "kl")])
def test_1vsall_job_on_wrapper(base, loss, dropout, subbatch, splits, stub):
    out = _pair(base, "1vsAll", loss, "B200TrainingJob1vsAll", splits, dropout=dropout, subbatch=subbatch)
    assert calls and all(c[0] == "1vsall" and c[1] == R and c[2] == dropout for c in calls)
    assert out["plugin"] == pytest.approx(out["ref"], rel=REL)


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("loss,eps", [("kl", 0.0), ("bce", 0.1)])
def test_kvsall_job_on_wrapper(loss, eps, dropout, splits, stub):
    out = _pair("complex", "KvsAll", loss, "B200TrainingJobKvsAll", splits, extra={"KvsAll.label_smoothing": eps},
                dropout=dropout)
    assert out["plugin"] == pytest.approx(out["ref"], rel=REL)
    # both query types run as sp_ folds; the _po type's relation rows are p + R and, under dropout, its streams _po
    assert calls and all(c[1] == "sp_" for c in calls)
    po = [c for c in calls if c[4] == "_po" or (not dropout and bool((c[3] >= R).all()))]
    assert po and all(bool((c[3] >= R).all()) for c in po)
    assert any(bool((c[3] < R).all()) and c[4] is None for c in calls)
    if dropout:
        assert all(c[4] == "_po" for c in calls if bool((c[3] >= R).all()))


@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("base", ["complex", "transe"])
def test_negative_sampling_job_on_wrapper(base, impl, splits, stub):
    extra = {"negative_sampling.implementation": impl, "negative_sampling.num_samples.s": 3,
             "negative_sampling.num_samples.o": 4}
    seen = []
    from kge_b200.plugin import _B200ModelMixin

    orig = _B200ModelMixin.loss_negatives

    def record(self, triples, negatives, slot, *a, **kw):
        seen.append((triples.clone(), slot))
        return orig(self, triples, negatives, slot, *a, **kw)
    _B200ModelMixin.loss_negatives = record
    try:
        out = _pair(base, "negative_sampling", "bce", "B200TrainingJobNegativeSampling", splits, extra=extra)
    finally:
        _B200ModelMixin.loss_negatives = orig
    assert out["plugin"] == pytest.approx(out["ref"], rel=REL)
    # every call runs the O-slot kernels; the S slot's triples are (o, p + R, s)
    assert seen and all(slot == 2 for _, slot in seen)
    assert any(bool((t[:, 1] >= R).all()) for t, _ in seen) and any(bool((t[:, 1] < R).all()) for t, _ in seen)


def _ran_reference(job):
    job.epoch += 1
    job._prepare()
    job.run_epoch()
    return not calls


def test_non_b200_base_falls_through(splits, stub):
    assert _ran_reference(_make("complex", "1vsAll", "kl", splits, "B200TrainingJob1vsAll"))


def test_s_o_query_type_falls_through(splits, stub):
    job = _make("b200_complex", "KvsAll", "kl", splits, "B200TrainingJobKvsAll", {"KvsAll.query_types.s_o": True})
    with pytest.raises(Exception):       # the reference wrapper cannot score relations
        job.epoch += 1
        job._prepare()
        job.run_epoch()
    assert not calls


@pytest.mark.parametrize("extra", [{"negative_sampling.num_samples.p": 2},
                                   {"b200_complex.entity_embedder.dropout": 0.3, "user.b200_ns_dropout": True}])
def test_ns_p_slot_and_dropout_keep_todays_route(extra, splits, stub):
    job = _make("b200_complex", "negative_sampling", "kl", splits, "B200TrainingJobNegativeSampling", extra)
    base = job.model._base_model
    ran = []
    base.loss_negatives = lambda *a, **kw: ran.append(1)
    base.score_negatives = lambda *a, **kw: ran.append(1)
    job.epoch += 1
    job._prepare()
    try:
        job.run_epoch()
    except Exception:                    # the reference raises for the P slot of the wrapper
        pass
    assert not ran


def test_ns_device_sampling_names_the_reason(splits, stub):
    job = _make("b200_complex", "negative_sampling", "kl", splits, "B200TrainingJobNegativeSampling",
                {"negative_sampling.num_samples.p": 2, "user.b200_device_sampling": True})
    job.epoch += 1
    job._prepare()
    with pytest.raises(NotImplementedError, match="reciprocal_relations_model: the P slot"):
        job.run_epoch()
