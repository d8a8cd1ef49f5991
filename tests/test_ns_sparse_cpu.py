"""Row-sparse table gradients of the negative-sampling step without a GPU: the row-set mirror against LibKGE's own
nn.Embedding(sparse=True) lookups, the argument checks and workspace size of b200kge_ns_backward_sparse, the routing
of `lookup_embedder.sparse`, and two epochs of the plugin job against the reference job with sparse gradients."""
import ctypes as C

import numpy as np
import pytest
import torch

import ns_loss_oracle as nlo
import ns_sparse_oracle as nsp
from kge_b200 import hostenv

S, P, O = 0, 1, 2


def _reference_lookups(tri, neg, slot, impl, E, R, D=4):
    """The rows nn.Embedding(sparse=True) reports after the reference's lookups of one slot (sampler.py:263-344 and the
    positive's score_spo, train_negative_sampling.py:139-148)."""
    ent, rel = torch.nn.Embedding(E, D, sparse=True), torch.nn.Embedding(R, D, sparse=True)
    out = ent(tri[:, 0]).sum() + rel(tri[:, 1]).sum() + ent(tri[:, 2]).sum()
    if impl == "triple":
        t = tri.repeat(1, neg.shape[1]).view(-1, 3)
        t[:, slot] = neg.reshape(-1)
        out = out + ent(t[:, 0]).sum() + rel(t[:, 1]).sum() + ent(t[:, 2]).sum()
    else:
        fixed = 2 if slot == S else 0
        out = out + ent(tri[:, fixed]).sum() + rel(tri[:, 1]).sum()
        out = out + (ent(torch.arange(E)) if impl == "all" else ent(torch.unique(neg))).sum()
    out.backward()
    return (ent.weight.grad.coalesce().indices()[0].numpy(), rel.weight.grad.coalesce().indices()[0].numpy())


@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
@pytest.mark.parametrize("slot", [S, O])
def test_row_set_mirror_matches_reference_lookups(impl, slot):
    g = torch.Generator().manual_seed(slot + 7)
    E, R, n, K = 30, 4, 5, 6
    tri = torch.stack([torch.randint(0, E, (n,), generator=g), torch.randint(0, R, (n,), generator=g),
                       torch.randint(0, E, (n,), generator=g)], 1)
    neg = torch.randint(0, E, (n, K), generator=g)
    neg[:, 1] = neg[:, 2]                       # repeated ids
    tri[1] = tri[0]
    want = _reference_lookups(tri, neg, slot, impl, E, R)
    got = nsp.row_sets(tri.numpy(), neg.numpy(), impl, E)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


# ---- C ABI: argument checks (all before any launch) and the workspace size
@pytest.fixture(scope="module")
def lib():
    from kge_b200 import _lib

    try:
        return _lib.load()
    except OSError as e:
        pytest.skip(f"libb200kge.so not loadable here: {e}")


def _call(lib, **over):
    from kge_b200._lib import Rows

    E, R, D, n, K = 50, 6, 16, 3, 4
    buf = (C.c_float * 16)()
    ids = (C.c_int64 * 64)()
    ent, rel = Rows(), Rows()
    for r, rows in ((ent, E), (rel, R)):
        r.base, r.idx, r.rows, r.ld, r.dim = C.addressof(buf), None, rows, D, D
    a = dict(model=0, l_norm=1.0, ent=ent, rel=rel, triples=C.addressof(ids), slot=2, neg=C.addressof(ids), n=n, K=K,
             impl=0, drop=None, g=None, ldg=0, offset=0.0, bs=n, es=1, er=C.addressof(ids), ec=C.addressof(ids),
             de=C.addressof(buf), lde=D, rs=1, rr=C.addressof(ids), rcnt=C.addressof(ids), dr=C.addressof(buf), ldr=D,
             ws=C.addressof(buf), wsb=0)
    a.update(over)
    return lib.b200kge_ns_backward_sparse(a["model"], a["l_norm"], C.byref(a["ent"]), C.byref(a["rel"]), a["triples"],
                                          a["slot"], a["neg"], a["n"], a["K"], a["impl"], a["drop"], a["g"], a["ldg"],
                                          a["offset"], a["bs"], a["es"], a["er"], a["ec"], a["de"], a["lde"], a["rs"],
                                          a["rr"], a["rcnt"], a["dr"], a["ldr"], a["ws"], a["wsb"], None)


def test_sparse_entry_refuses_bad_arguments(lib):
    from kge_b200._lib import ERR_INVALID as INVALID, ERR_UNSUPPORTED as UNSUPPORTED, ERR_WORKSPACE as WORKSPACE

    assert _call(lib, triples=None) == INVALID
    assert _call(lib, er=None) == INVALID                       # sparse entity table without rows
    assert _call(lib, rcnt=None) == INVALID                     # sparse relation table without a count
    assert _call(lib, de=None) == INVALID
    assert _call(lib, bs=0) == INVALID
    assert _call(lib, lde=8) == INVALID
    assert _call(lib, n=-1) == INVALID
    assert _call(lib, slot=1) == UNSUPPORTED
    assert _call(lib, model=5, l_norm=3.0) in (INVALID, UNSUPPORTED)
    assert _call(lib, wsb=0) == WORKSPACE
    assert _call(lib, ws=None, wsb=1 << 20) == WORKSPACE
    # without a sparse table the row outputs may be null, like the dense entry's
    assert _call(lib, es=0, er=None, ec=None, rs=0, rr=None, rcnt=None, wsb=0) == WORKSPACE


def test_sparse_entry_workspace_bytes(lib):
    def up(b):
        return (b + 255) // 256 * 256

    for model, n, K, D, E, R, drop in ((0, 3, 4, 16, 50, 6, 0), (1, 512, 1000, 512, 40943, 237, 1),
                                       (0, 512, 1000, 512, 4_800_000, 822, 0), (6, 7, 2, 64, 1, 1, 1)):
        rows = sum(up(V * 4) + up(-(-V // 4096) * 4) for V in (E, R))
        dense = lib.b200kge_ns_backward_workspace_bytes(model, n, K, D, drop)
        assert lib.b200kge_ns_backward_sparse_workspace_bytes(model, n, K, D, E, R, drop) == rows + up(dense)
    assert lib.b200kge_ns_backward_sparse_workspace_bytes(0, -1, 4, 16, 50, 6, 0) == 0


# ---- the job on the CPU (engine stand-ins): routing and two epochs against the reference job
E, R, D = 30, 4, 8


@pytest.fixture()
def splits():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 120, 20, 20)


@pytest.fixture()
def stub():
    """tests/engine_stub.py plus oracle-backed ns_loss, the grad_scores form of ns_backward and ns_backward_sparse (the
    dense oracle gradient restricted to the mirror's row set); counts the backward calls."""
    import engine_stub
    from kge_b200 import engine
    from oracle import kge_fold as kf

    calls = {"ns_backward": 0, "ns_backward_sparse": 0}
    plain = engine_stub.ns_backward

    def ns_loss(scores, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None, want_grad=False,
                return_rows=False):
        z = scores.detach()
        return (nlo.ns_loss(z, loss, arg, temperature, label_idx, batch_size),
                nlo.ns_loss_grad(z, loss, arg, temperature, label_idx, batch_size) if want_grad else None)

    def dense(model, ent, rel, triples, negatives, offset, l_norm, batch_size, grad_scores):
        if grad_scores is None:
            return plain(model, ent, rel, triples, negatives, offset, l_norm, batch_size)
        d_ent, d_rel = torch.zeros_like(ent), torch.zeros_like(rel)
        n = triples.shape[0]
        for slot, neg in negatives.items():
            k = neg.shape[1]
            t = triples.long().repeat_interleave(1 + k, 0).view(n, 1 + k, 3).clone()
            t[:, 1:, slot] = neg.long()
            t = t.view(-1, 3)
            kf.spo_backward(model, ent.detach(), rel.detach(), t[:, 0], t[:, 1], t[:, 2],
                            grad_scores[slot].reshape(-1), d_ent, d_rel, l_norm)
        return d_ent, d_rel

    def ns_backward(model, ent, rel, triples, negatives, offset=0.0, l_norm=1.0, batch_size=None, grad_scores=None):
        calls["ns_backward"] += 1
        return dense(model, ent, rel, triples, negatives, offset, l_norm, batch_size, grad_scores)

    def ns_backward_sparse(model, ent, rel, triples, slot, negatives, offset=0.0, l_norm=1.0, batch_size=None,
                           grad_scores=None, dropout=None, implementation="batch", sparse=(True, True)):
        assert dropout is None
        calls["ns_backward_sparse"] += 1
        d = dense(model, ent, rel, triples, {slot: negatives}, offset, l_norm, batch_size,
                  None if grad_scores is None else {slot: grad_scores})
        rows = nsp.row_sets(triples.numpy(), negatives.numpy(), implementation, ent.shape[0])
        out = []
        for x, r, sp in zip(d, rows, sparse):
            r = torch.from_numpy(r)
            out.append(torch.sparse_coo_tensor(r[None, :], x[r], x.shape, is_coalesced=True) if sp else x)
        return tuple(out)

    with engine_stub.installed():
        saved = engine.ns_loss, engine.ns_backward, engine.ns_backward_sparse
        engine.ns_loss, engine.ns_backward, engine.ns_backward_sparse = ns_loss, ns_backward, ns_backward_sparse
        try:
            yield calls
        finally:
            engine.ns_loss, engine.ns_backward, engine.ns_backward_sparse = saved


def _record_layouts(job):
    """The layout of every parameter's .grad at each optimizer step (before the step and its zero_grad)."""
    seen = []
    step = job.optimizer.step

    def recording_step(*a, **kw):
        seen.append(tuple(p.grad is not None and p.grad.is_sparse for p in job.model.parameters()))
        return step(*a, **kw)
    job.optimizer.step = recording_step
    return seen


def _pair(splits, loss, optimizer, impl, sparse_ent=True, sparse_rel=True):
    import jobs_util as ju

    torch.manual_seed(0)
    extra = {"negative_sampling.num_samples.s": 4, "negative_sampling.num_samples.o": 5,
             "negative_sampling.implementation": impl, "train.optimizer.default.type": optimizer,
             "train.loss_arg": 1.0 if loss == "bce" else 0.5,
             "complex.entity_embedder.sparse": sparse_ent, "complex.relation_embedder.sparse": sparse_rel}
    init = ju.make_job("complex", E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=16, extra=extra)
    jobs = {}
    for tag in ("ref", "plugin"):
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "plugin" else {}
        ex = dict(extra)
        if tag == "plugin":
            ex = {k.replace("complex.", "b200_complex."): v for k, v in ex.items()}
        jobs[tag] = ju.make_job("complex" if tag == "ref" else "b200_complex", E, R, D, splits,
                                train_type="negative_sampling", loss=loss, batch_size=16, forward_only=False, extra=ex,
                                **kw)
        ju.copy_tables(init, jobs[tag])
    return jobs


def _epochs(job, n=2):
    import jobs_util as ju

    out = []
    for ep in range(n):
        job.epoch += 1
        if job.loader is None:
            job._prepare()
        ju.seed_all(10 + ep)
        out.append(job.run_epoch()["avg_loss"])
    return out


def test_dense_tables_keep_the_dense_route(splits, stub):
    jobs = _pair(splits, "kl", "Adagrad", "batch", False, False)
    _epochs(jobs["plugin"], 1)
    assert stub["ns_backward"] > 0 and stub["ns_backward_sparse"] == 0, stub


@pytest.mark.parametrize("sparse", [(True, False), (False, True)])
def test_either_sparse_table_takes_the_sparse_route(splits, stub, sparse):
    jobs = _pair(splits, "kl", "Adagrad", "batch", *sparse)
    _epochs(jobs["plugin"], 1)
    assert stub["ns_backward"] == 0 and stub["ns_backward_sparse"] > 0, stub


@pytest.mark.parametrize("loss", ["kl", "bce"])
@pytest.mark.parametrize("optimizer", ["Adagrad", "SparseAdam"])
@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
def test_two_epochs_match_reference(splits, stub, loss, optimizer, impl):
    jobs = _pair(splits, loss, optimizer, impl)
    seen = {tag: _record_layouts(job) for tag, job in jobs.items()}
    out = {tag: _epochs(job) for tag, job in jobs.items()}
    assert stub["ns_backward_sparse"] > 0
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)
    for tag in jobs:                        # both tables row-sparse at every step, in both jobs
        assert seen[tag] and all(all(layout) for layout in seen[tag]), (tag, seen[tag][:3])
    w = [job.model.get_s_embedder()._embeddings.weight.detach() for job in jobs.values()]
    assert torch.allclose(w[0], w[1], rtol=1e-5, atol=1e-6)


def test_grad_is_sparse_after_backward(splits, stub):
    jobs = _pair(splits, "kl", "Adagrad", "batch")
    job = jobs["plugin"]
    job._prepare()
    tri = job.dataset.split("train")[:8].long()
    negs = torch.randint(0, E, (8, 5))
    loss = job.model.loss_negatives(tri, negs, O, 0.5, 8, "kl")
    loss.backward()
    w_e, w_r = job.model._b200_weights()
    assert w_e.grad.is_sparse and w_r.grad.is_sparse
    rows = nsp.row_sets(tri.numpy(), negs.numpy(), "batch", E)
    assert torch.equal(w_e.grad.coalesce().indices()[0], torch.from_numpy(rows[0]))


def test_adam_raises_like_the_reference(splits, stub):
    jobs = _pair(splits, "kl", "Adam", "batch")
    errors = {}
    for tag, job in jobs.items():
        with pytest.raises(RuntimeError) as e:
            _epochs(job, 1)
        errors[tag] = (type(e.value), str(e.value))
    assert errors["ref"] == errors["plugin"]
    assert "does not support sparse gradients" in errors["plugin"][1]


def test_reciprocal_job_relation_rows_and_epochs(splits, stub, monkeypatch):
    """The reciprocal wrapper's S slot goes through the O-slot backward as (o, p + R, s'): its relation rows are p + R
    of the 2R-row table; two epochs match the reference wrapper with sparse gradients."""
    import jobs_util as ju
    from kge_b200 import engine

    calls = []
    inner = engine.ns_backward_sparse

    def spy(model, ent, rel, triples, slot, negatives, *a, **kw):
        out = inner(model, ent, rel, triples, slot, negatives, *a, **kw)
        calls.append((slot, triples.clone(), rel.shape[0], out[1].coalesce().indices()[0].clone()))
        return out
    monkeypatch.setattr(engine, "ns_backward_sparse", spy)
    torch.manual_seed(0)
    extra = {"negative_sampling.num_samples.s": 4, "negative_sampling.num_samples.o": 5,
             "negative_sampling.implementation": "batch", "train.optimizer.default.type": "SparseAdam",
             "lookup_embedder.sparse": True}

    def make(base, **kw):
        ex = dict(extra, **{"reciprocal_relations_model.base_model.type": base})
        return ju.make_job("reciprocal_relations_model", E, R, D, splits, train_type="negative_sampling", loss="kl",
                           batch_size=16, extra=ex, imports=(base,), **kw)
    init = make("complex")
    jobs = {"ref": make("complex", forward_only=False),
            "plugin": make("b200_complex", forward_only=False, job_class="B200TrainingJobNegativeSampling")}
    seen = {}
    for job in jobs.values():
        ju.copy_tables(init, job)
    for tag, job in jobs.items():
        seen[tag] = _record_layouts(job)
    out = {tag: _epochs(job) for tag, job in jobs.items()}
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)
    for tag in jobs:
        assert seen[tag] and all(all(layout) for layout in seen[tag]), (tag, seen[tag][:3])
    s_calls = [c for c in calls if int(c[1][:, 1].min()) >= R]
    o_calls = [c for c in calls if int(c[1][:, 1].max()) < R]
    assert s_calls and o_calls and len(s_calls) + len(o_calls) == len(calls)
    for slot, tri, rows, rel_rows in calls:
        assert slot == O and rows == 2 * R
        assert torch.equal(rel_rows, torch.unique(tri[:, 1]))
