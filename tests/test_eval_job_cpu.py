"""Host logic of B200EntityRankingJob on CPU: routing through the reference's job factory, the collate's CSR filters,
the traces against the unmodified EntityRankingJob, and the tie-handling check.  kge_b200.engine is replaced by the
oracle-backed stand-in of tests/engine_stub.py plus, below, a stand-in of engine.rank_sp_po_eval that ranks the oracle's
dense scores with the filters densified (the kernel itself is tested in tests/test_gpu_eval_job.py)."""
import pytest
import torch

from kge_b200 import hostenv

pytestmark = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")

import engine_stub  # noqa: E402
import jobs_util as ju  # noqa: E402
from oracle import kge_oracle as orc  # noqa: E402

E, R, D = 53, 4, 16
CLS = {"entity_ranking.class_name": "B200EntityRankingJob"}
_IDS = ("epoch_time", "timestamp", "job_id", "parent_job_id", "entry_id")   # differ between any two runs


@pytest.fixture(scope="module")
def splits():
    return ju.synthetic_splits(E, R, 150, 20, 20)


def _densify(off, col, own, m):
    n2 = off.numel() - 1
    lab = torch.zeros((n2, m))
    rows = torch.repeat_interleave(torch.arange(n2), off[1:] - off[:-1])
    lab[rows, col.long()] = float("inf")
    lab[torch.arange(n2), own.long()] = 0.0
    return lab


_perturb = {"own": 0.0}


def rank_sp_po_eval(model, ent, rel, s, p, o, true_scores, own_col, filter_off, filter_col, test_off=None,
                    test_col=None, rtol=1e-4, atol=1e-5, l_norm=1.0, precision="auto", num_relations=0):
    engine_stub._counter["n"] += 1
    s, p, o = s.long(), p.long(), o.long()
    n = s.numel()
    if num_relations:
        x = torch.cat((orc.score_sp(model, ent, rel, s, p, None, l_norm),
                       orc.score_sp(model, ent, rel, o, p + num_relations, None, l_norm)))
    else:
        y = orc.score_sp_po(model, ent, rel, s, p, o, None, l_norm)
        x = torch.cat((y[:, :E], y[:, E:]))
    own = own_col.long()
    own_score = x[torch.arange(2 * n), own] + _perturb["own"]
    t = true_scores.reshape(-1)
    counts = [orc.ranks_and_ties(x, t, rtol, atol)]
    x = x - _densify(filter_off, filter_col, own, E)
    counts.append(orc.ranks_and_ties(x, t, rtol, atol))
    if test_off is not None:
        x = x - _densify(test_off, test_col, own, E)
        counts.append(orc.ranks_and_ties(x, t, rtol, atol))
    return torch.stack([c[0] for c in counts]), torch.stack([c[1] for c in counts]), own_score


@pytest.fixture()
def stub():
    from kge_b200 import engine

    saved = engine.rank_sp_po_eval
    with engine_stub.installed():
        engine.rank_sp_po_eval = rank_sp_po_eval
        try:
            yield
        finally:
            engine.rank_sp_po_eval = saved
            _perturb["own"] = 0.0


def _job(model, splits, extra=None, imports=(), cls=True):
    torch.manual_seed(0)
    cfg = dict(CLS if cls else {}, **(extra or {}))
    return ju.make_job(model, E, R, D, splits, loss="kl", batch_size=32, extra=cfg, imports=imports)


def _traces(job):
    """(epoch trace, every trace entry the validation job wrote) of one validation run."""
    ev = job.valid_job
    entries = []
    orig = ev.trace

    def trace(**kw):
        entries.append({k: v for k, v in kw.items() if k != "epoch_time"})
        return orig(**kw)
    ev.trace = trace
    out = ju.run_valid(job)
    return {k: v for k, v in out.items() if k not in _IDS}, entries


def _same(a, b):
    """dict equality with NaN equal to NaN (valid.metric_expr yields NaN for a metric the run did not compute)"""
    def eq(x, y):
        return x == y or (isinstance(x, float) and isinstance(y, float) and x != x and y != y)
    return a.keys() == b.keys() and all(eq(a[k], b[k]) for k in a)


def _compare(model, splits, extra=None, imports=()):
    ref = _job(model, splits, extra, imports, cls=False)
    fused = _job(model, splits, extra, imports)
    ju.copy_tables(ref, fused)
    assert type(fused.valid_job).__name__ == "B200EntityRankingJob"
    assert type(ref.valid_job).__name__ == "EntityRankingJob"
    engine_stub.launch_count(reset=True)
    a, ea = _traces(ref)
    b, eb = _traces(fused)
    assert fused.valid_job._b200_route is not None
    assert _same(a, b)
    assert len(ea) == len(eb) and all(_same(x, y) for x, y in zip(ea, eb))
    return fused, b, eb


@pytest.mark.parametrize("tie", ["rounded_mean_rank", "best_rank", "worst_rank"])
@pytest.mark.parametrize("with_test", [True, False])
def test_traces_equal_reference(tie, with_test, splits, stub):
    extra = {"entity_ranking.tie_handling.type": tie, "entity_ranking.filter_with_test": with_test,
             "valid.trace_level": "example", "eval.batch_size": 7}
    fused, b, entries = _compare("b200_complex", splits, extra)
    assert ("hits_at_1_filtered_with_test" in b) == with_test
    assert sum(e.get("event") == "example_rank" for e in entries) == 2 * len(splits["valid"])
    assert sum(e.get("scope") == "batch" for e in entries) == len(fused.valid_job.loader)


def test_test_split_and_metrics_per(splits, stub):
    extra = {"valid.split": "test", "entity_ranking.filter_with_test": True, "train.trace_level": "batch",
             "entity_ranking.metrics_per.relation_type": True, "entity_ranking.metrics_per.head_and_tail": True,
             "entity_ranking.metrics_per.argument_frequency": True}
    _, b, _ = _compare("b200_transe", splits, extra)
    assert "mean_reciprocal_rank_filtered_head" in b and "hits_at_1_filtered_tail" in b


@pytest.mark.parametrize("base", ["b200_complex", "b200_cp"])
def test_reciprocal_wrapper(base, splits, stub):
    extra = {"reciprocal_relations_model.base_model.type": base, "entity_ranking.filter_with_test": True}
    fused, _, _ = _compare("reciprocal_relations_model", splits, extra, imports=(base,))
    assert fused.valid_job._b200_route[1] == R


def test_one_rank_call_per_batch(splits, stub):
    job = _job("b200_distmult", splits, {"entity_ranking.filter_with_test": True})
    engine_stub.launch_count(reset=True)
    ju.run_valid(job)
    # per batch: score_sp and score_po for the true scores, then ONE ranking call
    assert engine_stub.launch_count() == 3 * len(job.valid_job.loader)


def test_routing_falls_through(splits, stub):
    """A non-b200 model or an in-kernel split precision runs the reference's _evaluate, with no ranking call."""
    for model, extra in (("distmult", {}), ("b200_distmult", {"b200_distmult.precision": "tf32"})):
        ref = _job("distmult", splits, cls=False)
        job = _job(model, splits, extra)
        ju.copy_tables(ref, job)
        engine_stub.launch_count(reset=True)
        b = ju.run_valid(job)
        assert type(job.valid_job).__name__ == "B200EntityRankingJob" and job.valid_job._b200_route is None
        if model == "distmult":
            assert engine_stub.launch_count() == 0
        a = ju.run_valid(ref)
        assert b["mean_reciprocal_rank_filtered"] == pytest.approx(a["mean_reciprocal_rank_filtered"], rel=1e-5)


def test_routing_separate_embedders(splits, stub):
    """Separate subject and object embedders: the tables cannot be read in place, the reference's _evaluate runs."""
    import copy

    job = _job("b200_distmult", splits)
    other = copy.deepcopy(job.model.get_o_embedder())
    job.model.get_o_embedder = lambda: other
    job.model.__dict__.pop("_b200_fusable_cache", None)
    job.valid_job._prepare()
    assert job.valid_job._b200_route is None


def test_collate_matches_reference_coordinates(splits, stub):
    import kge.job.util as ku

    job = _job("b200_simple", splits, {"entity_ranking.filter_with_test": True})
    ev = job.valid_job
    ev._prepare()
    ds = ev.dataset
    rows = [t for t in ds.split("valid")[:13]]
    batch, (f_off, f_col), (t_off, t_col), own = ev._collate(rows)
    n = len(rows)
    assert torch.equal(own, torch.cat((batch[:, 2], batch[:, 0])).long())

    def coords_set(split_names):
        cs = torch.cat([ku.get_sp_po_coords_from_spo_batch(batch, E, ds.index(f"{sp}_sp_to_o"), ds.index(f"{sp}_po_to_s"))
                        for sp in split_names]).long()
        # reference layout: [n, 2E]; ours: rows [0, n) sp_, rows [n, 2n) _po
        return {(int(r) + (n if c >= E else 0), int(c) % E) for r, c in cs.tolist()}

    def csr_set(off, col):
        for r in range(2 * n):
            seg = col[off[r]:off[r + 1]]
            assert torch.equal(seg, torch.unique(seg))          # sorted and unique
        rows = torch.repeat_interleave(torch.arange(2 * n), off[1:] - off[:-1])
        return set(zip(rows.tolist(), col.tolist()))

    F = csr_set(f_off, f_col)
    T = csr_set(t_off, t_col)
    assert F == coords_set(ev.filter_splits)
    assert not (F & T)
    assert T == coords_set(["test"]) - F


def test_tie_check(splits, stub, capsys):
    job = _job("b200_rescal", splits, {"entity_ranking.tie_handling.warn_only": False})
    _perturb["own"] = 1.0
    with pytest.raises(ValueError, match="tie-handling"):
        ju.run_valid(job)
    job = _job("b200_rescal", splits, {"entity_ranking.tie_handling.warn_only": True})
    out = ju.run_valid(job)
    assert "mean_reciprocal_rank_filtered" in out
    assert "tie-handling" in capsys.readouterr().err
