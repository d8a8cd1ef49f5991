"""b200kge_rank_sp_po_eval (every ranking of an evaluation batch from one scoring pass) against the existing kernels,
bit for bit, and B200EntityRankingJob against the unmodified EntityRankingJob on the same plugin model."""
import pytest
import torch

from kge_b200 import engine, hostenv
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

E_, R_, D_ = 5003, 11, 128
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]


def _csr(lists):
    off = torch.zeros(len(lists) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor([len(x) for x in lists]), 0)
    col = torch.tensor([c for x in lists for c in sorted(x)], dtype=torch.int64)
    return off, col


def _dense(lists, own, m):
    f = torch.zeros((len(lists), m))
    for r, x in enumerate(lists):
        for c in x:
            f[r, c] = float("inf")
        f[r, own[r]] = 0.0
    return f


def _filters(own, m, g):
    """F (lists that contain the own column, span tiles or are empty) and T' (disjoint from F) per stacked row."""
    F, T = [], []
    for r, a in enumerate(own.tolist()):
        kind = r % 4
        f = set() if kind == 0 else set(torch.randint(0, m, (int(torch.randint(1, 60, (1,), generator=g)),),
                                                      generator=g).tolist())
        if kind in (1, 3):
            f.add(a)
        if kind == 2:
            f |= {a - 1 if a > 0 else a + 1, (a + 128) % m, (a + 300) % m}
        t = set(torch.randint(0, m, (int(torch.randint(0, 20, (1,), generator=g)),), generator=g).tolist()) - f - {a}
        F.append(f)
        T.append(t)
    return F, T


@pytest.mark.parametrize("model,ln", CASES)
@pytest.mark.parametrize("n,precision", [(40, "auto"), (9, "auto"), (70, "fp32")])
@pytest.mark.parametrize("recip", [False, True])
def test_entry_bit_exact(model, ln, n, precision, recip):
    g = torch.Generator().manual_seed(n + 7 * len(model))
    R = 2 * R_ if recip else R_
    ent, rel = orc.make_tables(model, E_, R, D_, sigma=0.5)
    ent, rel = ent.cuda(), rel.cuda()
    tri = orc.make_triples(E_, R_, n, seed=n).cuda()
    s, p, o = tri[:, 0], tri[:, 1], tri[:, 2]
    # the stored scores of both halves (sp_ rows, then _po rows or the reciprocal sp_ rows (o, p + R_))
    x1 = engine.score_1vsN(model, "sp_", ent, rel, ent, s, p, None, ln, precision)
    x2 = (engine.score_1vsN(model, "sp_", ent, rel, ent, o, p + R_, None, ln, precision) if recip else
          engine.score_1vsN(model, "_po", ent, rel, ent, o, p, None, ln, precision))
    X = torch.cat((x1, x2))
    own = torch.cat((o, s))
    rows = torch.arange(2 * n, device="cuda")
    t = X[rows, own].clone()
    t[1::5] += 1e-3                       # true scores that tie with nothing / with neighbours
    t[3], t[5], t[7] = float("nan"), float("-inf"), float("inf")
    F, T = _filters(own.cpu(), E_, g)
    FT = [a | b for a, b in zip(F, T)]
    f_off, f_col = (z.cuda() for z in _csr(F))
    t_off, t_col = (z.cuda() for z in _csr(T))
    rank, ties, own_score = engine.rank_sp_po_eval(model, ent, rel, s, p, o, t, own, f_off, f_col, t_off, t_col,
                                                   1e-4, 1e-5, ln, precision, num_relations=R_ if recip else 0)
    torch.cuda.synchronize()
    assert torch.equal(own_score, X[rows, own])
    want = [engine.rank_dense(X, t),
            engine.rank_dense(X, t, _dense(F, own.tolist(), E_).cuda()),
            engine.rank_dense(X, t, _dense(FT, own.tolist(), E_).cuda())]
    for k, (r, c) in enumerate(want):
        assert torch.equal(rank[k], r), k
        assert torch.equal(ties[k], c), k
    if model != "cp" and not recip:
        r, c = engine.rank_sp_po_csr(model, ent, rel, ent, ent, t, f_off, f_col, own, s, p, o, 1e-4, 1e-5, ln, precision)
        assert torch.equal(rank[1], r) and torch.equal(ties[1], c)
        r, c = engine.rank_sp_po(model, ent, rel, ent, ent, t, s, p, o, None, None, 1e-4, 1e-5, ln, precision)
        assert torch.equal(rank[0], r) and torch.equal(ties[0], c)
    # without T': two rankings, the same counts
    rank2, ties2, _ = engine.rank_sp_po_eval(model, ent, rel, s, p, o, t, own, f_off, f_col, None, None, 1e-4, 1e-5, ln,
                                             precision, num_relations=R_ if recip else 0)
    assert rank2.shape[0] == 2 and torch.equal(rank2, rank[:2]) and torch.equal(ties2, ties[:2])


def test_entry_refuses_split_modes_and_bad_reciprocal():
    ent, rel = orc.make_tables("complex", 300, R_, 64)
    ent, rel = ent.cuda(), rel.cuda()
    tri = orc.make_triples(300, R_, 20).cuda()
    own = torch.cat((tri[:, 2], tri[:, 0]))
    off = torch.zeros(41, dtype=torch.int64, device="cuda")
    col = torch.zeros(0, dtype=torch.int64, device="cuda")
    t = torch.zeros(40, device="cuda")
    with pytest.raises(NotImplementedError):
        engine.rank_sp_po_eval("complex", ent, rel, tri[:, 0], tri[:, 1], tri[:, 2], t, own, off, col,
                               precision="3xtf32")
    with pytest.raises(ValueError):
        engine.rank_sp_po_eval("complex", ent, rel, tri[:, 0], tri[:, 1], tri[:, 2], t, own, off, col,
                               num_relations=R_)          # rel has R_ rows, not 2 R_


# ------------------------------------------------------------------------------------------------------------------
# the job

needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
MODELS = ["complex", "distmult", "simple", "cp", "rescal", "transe", "rotate"]
E, R, D = 211, 5, 32
METRICS = [k + s for s in ("", "_filtered", "_filtered_with_test")
           for k in ("mean_rank", "mean_reciprocal_rank", "hits_at_1", "hits_at_3", "hits_at_10")]
CLS = {"entity_ranking.class_name": "B200EntityRankingJob"}


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 600, 60, 60)


def _job(ju, model, splits, device, extra, imports=()):
    torch.manual_seed(0)
    return ju.make_job(model, E, R, D, splits, device=device, train_type="1vsAll", loss="kl", batch_size=64,
                       extra=dict({"entity_ranking.filter_with_test": True, "eval.batch_size": 24}, **extra),
                       imports=imports)


def _run_counted(ju, job):
    calls = {"rank": 0, "sp_po": 0}
    saved = engine.rank_sp_po_eval, engine.score_sp_po

    def rank(*a, **kw):
        calls["rank"] += 1
        return saved[0](*a, **kw)

    def sp_po(*a, **kw):
        calls["sp_po"] += 1
        return saved[1](*a, **kw)
    engine.rank_sp_po_eval, engine.score_sp_po = rank, sp_po
    try:
        engine.launch_count(reset=True)
        out = ju.run_valid(job)
        torch.cuda.synchronize()
        return out, calls, engine.launch_count()
    finally:
        engine.rank_sp_po_eval, engine.score_sp_po = saved


def _compare(model, splits, extra=None, imports=()):
    import jobs_util as ju

    extra = dict(extra or {})
    ref_extra = {k: v.replace("b200_", "") if isinstance(v, str) else v for k, v in extra.items()}
    ref = _job(ju, model.replace("b200_", ""), splits, "cpu", ref_extra, tuple(i.replace("b200_", "") for i in imports))
    plug = _job(ju, model, splits, "cuda", extra, imports)
    fused = _job(ju, model, splits, "cuda", dict(extra, **CLS), imports)
    ju.copy_tables(ref, plug)
    ju.copy_tables(ref, fused)
    assert type(fused.valid_job).__name__ == "B200EntityRankingJob"
    a = ju.run_valid(ref)
    b = ju.run_valid(plug)
    c, calls, launches = _run_counted(ju, fused)
    nb = len(fused.valid_job.loader)
    assert fused.valid_job._b200_route is not None
    assert calls == {"rank": nb, "sp_po": 0}
    assert launches <= 16 * nb       # score_sp + score_po (true scores) + the ranking entry, a few launches each
    for k in METRICS:
        assert c[k] == b[k], k                       # same arithmetic as the unmodified job on the plugin model
        assert c[k] == pytest.approx(a[k], rel=5e-3, abs=5e-3), k
    assert c["mean_reciprocal_rank_filtered"] == pytest.approx(a["mean_reciprocal_rank_filtered"], rel=2e-3)


@needs_ref
@pytest.mark.parametrize("model", MODELS)
def test_job_matches_unmodified_job(model, splits):
    _compare("b200_" + model, splits)


@needs_ref
@pytest.mark.parametrize("base", ["b200_complex", "b200_transe"])
def test_job_reciprocal_wrapper(base, splits):
    _compare("reciprocal_relations_model", splits, {"reciprocal_relations_model.base_model.type": base},
             imports=(base,))


@needs_ref
def test_validation_during_training(splits):
    """Two training epochs with valid.every: 1: the validation job is a B200EntityRankingJob and its metrics equal those
    of the unmodified EntityRankingJob on the trained model."""
    import jobs_util as ju
    from kge.job import EvaluationJob

    job = _job(ju, "b200_complex", splits, "cuda", dict(CLS, **{"valid.every": 1, "train.max_epochs": 2}))
    job.is_forward_only = False
    assert type(job.valid_job).__name__ == "B200EntityRankingJob"
    job.run()
    assert job.epoch == 2 and len(job.valid_trace) == 2
    last = job.valid_trace[-1]
    conf = job.valid_job.config.clone()
    conf.set("entity_ranking.class_name", "EntityRankingJob")
    ref = EvaluationJob.create(conf, job.dataset, parent_job=job, model=job.model)
    assert type(ref).__name__ == "EntityRankingJob"
    ref._prepare()
    b = ref._run()
    for k in METRICS:
        assert last[k] == b[k], k
