"""Parity tests of the callers and rows either side of the scorer (SURVEY 8f): the evaluation loop on the fused rank kernels, the reference jobs' traces re-derived on the validated
entry points, one negative-sampling training batch, the reciprocal-relations model, Lp/N3 penalties + row
normalisation, and the KvsAll losses with CSR multi-hot labels."""
import os

import numpy as np
import pytest
import torch

from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
S, P, O = 0, 1, 2
TOL = 1e-4


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    return engine


def _load(name):
    z = np.load(os.path.join(GOLDEN, name))
    return {k: torch.from_numpy(z[k]) if z[k].ndim else z[k].item() for k in z.files}


def _assert_close(got, ref, what, tol=TOL):
    got = got.detach().cpu().double()
    ref = ref.double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    err = float((got - ref).abs().max()) if ref.numel() else 0.0
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


@pytest.mark.parametrize("model", ["complex", "transe"])
def test_evaluator_on_gpu_matches_reference_job(model):
    """kge_b200.evaluate.EntityRankingEvaluator driving the fused rank kernels reproduces the reference
    EntityRankingJob's trace (host logic is covered on CPU by tests/test_evaluate_cpu.py; this adds the device
    side: chunked subsets, dense filter planes, accumulation into rank/ties).  To be promoted into
    tests/test_gpu_model.py once it has run green on the GPU."""
    from kge_b200 import KgeModel
    from kge_b200.evaluate import EntityRankingEvaluator

    g = _load(f"jobs_{model}.npz")
    E, D = g["ent"].shape
    m = KgeModel(model, E, g["rel"].shape[0], D).cuda()
    with torch.no_grad():
        m.get_s_embedder().weight.copy_(g["ent"].cuda())
        m.get_p_embedder().weight.copy_(g["rel"].cuda())
    for bs, chunk in ((16, -1), (100, 7)):
        ev = EntityRankingEvaluator(m, E, [g["train"], g["valid"]], g["test"], batch_size=bs, chunk_size=chunk,
                                    hits_at_k_s=(1, 3, 10), device="cuda")
        met = ev.evaluate(g["valid"])
        for suffix in ("", "_filtered", "_filtered_with_test"):
            for k in ("mean_rank", "mean_reciprocal_rank", "hits_at_1", "hits_at_3", "hits_at_10"):
                want = float(g["valid_" + k + suffix])
                assert abs(met[k + suffix] - want) <= 1e-6 * max(1.0, abs(want)), (k + suffix, met[k + suffix], want)


@pytest.mark.parametrize("model", ["complex", "transe"])
def test_job_traces_on_gpu(eng, model):
    """Job-level traces of the reference (tests/golden/jobs_*.npz) through validated entry points only: 1vsAll
    epoch loss, KvsAll epochs with multi-hot / smoothed labels.  Gated until it has run once on the GPU."""
    g = _load(f"jobs_{model}.npz")
    ent, rel, train = g["ent"].cuda(), g["rel"].cuda(), g["train"].long().cuda()
    E = ent.shape[0]
    for loss in ("bce", "kl"):
        got = float(eng.train_1vsall_forward(model, ent, rel, train, loss))
        want = float(g[f"avg_loss_{loss}"])
        assert abs(got - want) <= 1e-4 * abs(want), (loss, got, want)

    def examples(key_cols, val_col):
        keys, inv = torch.unique(train[:, key_cols], dim=0, return_inverse=True)
        labels = torch.zeros((keys.shape[0], E), device="cuda")
        labels.index_put_((inv, train[:, val_col]), torch.ones(len(train), device="cuda"), accumulate=True)
        return keys, labels

    sp_keys, sp_lab = examples([S, P], O)
    po_keys, po_lab = examples([P, O], S)
    n = sp_keys.shape[0] + po_keys.shape[0]
    for loss, eps in (("kl", 0.0), ("kl", 0.2), ("bce", 0.2)):
        lab = (lambda y: (1.0 - eps) * y + 1.0 / E) if eps > 0 else (lambda y: y)
        l_sp = eng.score_1vsN_loss(model, "sp_", ent, rel, ent, lab(sp_lab), sp_keys[:, 0].contiguous(),
                                   sp_keys[:, 1].contiguous(), None, loss, 0.0)
        l_po = eng.score_1vsN_loss(model, "_po", ent, rel, ent, lab(po_lab), po_keys[:, 1].contiguous(),
                                   po_keys[:, 0].contiguous(), None, loss, 0.0)
        got = (float(l_sp) + float(l_po)) / n
        want = float(g[f"kvsall_avg_loss_{loss}_{int(eps * 10)}"])
        assert abs(got - want) <= 1e-4 * abs(want), (loss, eps, got, want)


@pytest.mark.parametrize("model", ["complex", "rotate"])
def test_ns_job_batch_on_gpu(eng, model):
    g = _load(f"nsjob_{model}.npz")
    ent, rel, tri = g["ent"].cuda(), g["rel"].cuda(), g["triples"].long().cuda()
    n, off = tri.shape[0], float(g["offset"])
    total = 0.0
    for slot, nm in ((S, "s"), (P, "p"), (O, "o")):
        neg = g[f"neg_{nm}"].long().cuda()
        scores = eng.ns_score(model, ent, rel, tri, neg, slot, True)
        labels = torch.zeros_like(scores)
        labels[:, 0] = 1.0
        total += float(eng.loss_dense(scores, labels, "bce", off)) / n
    assert abs(total - float(g["avg_loss"])) <= 1e-4 * abs(float(g["avg_loss"])), (total, float(g["avg_loss"]))


@pytest.mark.parametrize("base", ["complex", "transe"])
def test_reciprocal_model_on_gpu(base):
    """kge_b200.ReciprocalRelationsModel (index arithmetic over validated `sp_` entry points) against the live
    reference's ReciprocalRelationsModel.  Gated until it has run once on the GPU."""
    from kge_b200 import ReciprocalRelationsModel

    g = _load(f"reciprocal_{base}.npz")
    E, D = g["ent"].shape
    R = int(g["num_relations"])
    m = ReciprocalRelationsModel(base, E, R, D).cuda()
    with torch.no_grad():
        m.get_s_embedder().weight.copy_(g["ent"].cuda())
        m.get_p_embedder().weight.copy_(g["rel2"].cuda())
    tri, sub = g["triples"].long().cuda(), g["subset"].long().cuda()
    s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
    _assert_close(m.score_spo(s, p, o, "o"), g["spo_o"], "spo o")
    _assert_close(m.score_spo(s, p, o, "s"), g["spo_s"], "spo s")
    _assert_close(m.score_sp(s, p), g["sp"], "sp")
    _assert_close(m.score_po(p, o), g["po"], "po")
    _assert_close(m.score_po(p, o, sub), g["po_subset"], "po subset")
    _assert_close(m.score_sp_po(s, p, o), g["sp_po"], "sp_po")
    _assert_close(m.score_sp_po(s, p, o, sub), g["sp_po_subset"], "sp_po subset")


def test_penalties_and_normalisation_golden(eng):
    """Row kernels for Lp / N3 penalties and normalisation against the live reference (penalties.npz)."""
    import sys
    sys.path.insert(0, GOLDEN)
    from gen_golden import PENALTY_CASES

    g = _load("penalties.npz")
    for tag, model, eo, ro in PENALTY_CASES:
        space = "complex" if model == "complex" else "euclidean"
        ent, rel, tri = g[f"{tag}_ent"].cuda(), g[f"{tag}_rel"].cuda(), g[f"{tag}_triples"].long().cuda()

        def pen(w, o, idx):
            return float(eng.lookup_penalty(w, o["regularize"], o["regularize_weight"], float(o["p"]), o["weighted"],
                                              idx if o["weighted"] else None, space))

        total = pen(rel, ro, tri[:, P])
        total += pen(ent, eo, tri[:, [S, O]]) if eo["weighted"] else 2.0 * pen(ent, eo, None)
        want = float(g[f"{tag}_total"])
        assert abs(total - want) <= 1e-5 * abs(want), (tag, total, want)
    for pn in (1, 2):
        w = g["normalize_in"].cuda().clone()
        eng.normalize_rows_(w, float(pn))
        assert torch.allclose(w.cpu(), g[f"normalize_p{pn}"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("model,D", [("complex", 128), ("distmult", 32), ("rescal", 24), ("cp", 64), ("transe", 64), ("rotate", 64)])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_loss_with_csr_labels(eng, model, D, loss):
    """KvsAll losses with CSR multi-hot labels (duplicates, empty rows, label smoothing) against the oracle on the
    densified label matrix; both directions."""
    E, R, n = 3001, 5, 200
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.3)
    tri = orc.make_triples(E, R, n)
    g = torch.Generator().manual_seed(3)
    counts = (torch.rand((n, E), generator=g) < 0.004).float()
    counts[torch.arange(n), tri[:, O]] += 1.0
    counts[5, int(tri[5, O])] += 1.0          # a duplicate triple: label 2
    counts[7] = 0.0                            # a row without labels
    rows, cols = torch.nonzero(counts, as_tuple=True)
    rep = counts[rows, cols].long()
    cols_rep = torch.repeat_interleave(cols, rep)
    rows_rep = torch.repeat_interleave(rows, rep)
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.bincount(rows_rep, minlength=n), 0)
    ce, cr = ent.cuda(), rel.cuda()
    off = 1.0 if loss == "bce" else 0.0
    fn = (lambda x, y: orc.bce_loss(x, y, off)) if loss == "bce" else orc.kl_loss
    dot = model in ("complex", "distmult", "rescal", "cp")
    for combine, qi, sc in (("sp_", tri[:, S], orc.score_sp(model, ent, rel, tri[:, S], tri[:, P])),
                            ("_po", tri[:, O], orc.score_po(model, ent, rel, tri[:, P], tri[:, O]))):
        for eps in ((0.0, 0.1) if dot else (0.0,)):
            lab = orc.kvsall_smooth_labels(counts, eps) if eps > 0 else counts
            ref = float(fn(sc, lab))
            got, rws = eng.score_1vsN_loss_csr(model, combine, ce, cr, ce, offs.cuda(), cols_rep.cuda(), qi.cuda(),
                                                 tri[:, P].cuda(), loss, off, eps, return_rows=True)
            assert abs(float(got) - ref) <= 1e-4 * abs(ref), (model, loss, combine, eps, float(got), ref)
            assert abs(float(rws.sum()) - ref) <= 1e-4 * abs(ref)


@pytest.mark.parametrize("model,D", [("complex", 128), ("distmult", 64), ("rescal", 40), ("simple", 64), ("transe", 64),
                                     ("rotate", 64), ("distmult", 16)])
def test_rank_with_csr_filter_is_bit_identical_to_dense_filter(eng, model, D):
    """Filtered ranking with the known answers as CSR (consumed by the epilogues' cursors: tensor-core kernels for the
    dot family, CUDA-core kernel for TransE / RotatE and for K < 32) against the same call with the reference's dense
    +inf label matrix (eval_entity_ranking.py:489-531,561-566):
    integer counts, bit-identical; the row's own answer stays in (:287-290); ragged tiles, empty rows, rows with
    many listed columns, chunked candidates."""
    E, R, n = 5003, 5, 150
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n).cuda()
    ce, cr = ent.cuda(), rel.cuda()
    s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
    both = torch.cat([s, o])
    x = eng.score_sp_po(model, ce, cr, s, p, o, both)
    ar = torch.arange(n, device="cuda")
    true2n = torch.cat([x[ar, n + ar], x[ar, 2 * n + ar]]).contiguous()
    g = torch.Generator().manual_seed(3)
    counts = torch.randint(0, 40, (2 * n,), generator=g)
    counts[5] = 0
    counts[7] = 900
    own = torch.cat([o, s]).cpu()
    cols, offs = [], [0]
    for r in range(2 * n):
        c = torch.randperm(E, generator=g)[: int(counts[r])]
        c = torch.unique(torch.cat([c, own[r:r + 1]]))          # sorted, contains the own answer
        cols.append(c)
        offs.append(offs[-1] + c.numel())
    cols, offs = torch.cat(cols), torch.tensor(offs)
    dense = torch.zeros((2 * n, E))
    for r in range(2 * n):
        dense[r, cols[offs[r]:offs[r + 1]]] = float("inf")
    dense[torch.arange(2 * n), own] = 0.0
    for lo, hi in ((0, E), (1000, 3333)):                          # whole table and one chunk of candidates
        cand = ce[lo:hi]
        keep = (cols >= lo) & (cols < hi)
        rows = torch.repeat_interleave(torch.arange(2 * n), offs[1:] - offs[:-1])
        coffs = torch.zeros(2 * n + 1, dtype=torch.int64)
        coffs[1:] = torch.cumsum(torch.bincount(rows[keep], minlength=2 * n), 0)
        r1, t1 = eng.rank_sp_po(model, ce, cr, ce, cand, true2n, s, p, o, None, dense[:, lo:hi].contiguous().cuda())
        r2, t2 = eng.rank_sp_po_csr(model, ce, cr, ce, cand, true2n, coffs.cuda(), (cols[keep] - lo).cuda(),
                                    (own - lo).cuda(), s, p, o)
        assert torch.equal(r1, r2) and torch.equal(t1, t2)
        if lo == 0:
            assert int(t2.min()) >= 1                               # the own answer is a tie of itself


def test_rank_csr_is_refused_where_no_kernel_consumes_it(eng):
    """CP's two directions read different table columns (no stacked launch): the CSR form answers
    NotImplementedError before anything is launched and the caller passes the dense filter instead."""
    ent, rel = orc.make_tables("cp", 500, 3, 32)
    tri = orc.make_triples(500, 3, 20).cuda()
    z = torch.zeros(41, dtype=torch.int64, device="cuda")
    with pytest.raises(NotImplementedError):
        eng.rank_sp_po_csr("cp", ent.cuda(), rel.cuda(), ent.cuda(), ent.cuda(), torch.zeros(40, device="cuda"), z, z[:0], None,
                           tri[:, 0].contiguous(), tri[:, 1].contiguous(), tri[:, 2].contiguous())


def test_device_uniform_sampler(eng):
    """b200kge_sample_uniform: bit-exact against the Python Philox4x32-10 mirror (integers), reproducible, range-correct,
    and uniform (chi-square over 64 bins at 1e6 draws)."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from philox_ref import sample_uniform

    for n, K, vocab, seed, off in ((3, 7, 14541, 1234, 0), (2, 5, 4800000, 2 ** 40 + 17, 99), (1, 1, 3, 7, 2 ** 33)):
        got = eng.sample_uniform(n, K, vocab, seed, off, "cuda").cpu().view(-1).tolist()
        assert got == sample_uniform(n, K, vocab, seed, off)
    a = eng.sample_uniform(1000, 1000, 40943, 5, 1, "cuda")
    b = eng.sample_uniform(1000, 1000, 40943, 5, 1, "cuda")
    c = eng.sample_uniform(1000, 1000, 40943, 5, 2, "cuda")
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert int(a.min()) >= 0 and int(a.max()) < 40943
    hist = torch.bincount((a.view(-1) * 64) // 40943, minlength=64).double()
    chi2 = float(((hist - hist.mean()) ** 2 / hist.mean()).sum())
    assert chi2 < 120.0, chi2                                  # 63 dof: mean 63, p(chi2 > 120) ~ 1e-5


@pytest.mark.skipif(not __import__("kge_b200.hostenv", fromlist=["x"]).available(), reason="reference not installed")
def test_negative_sampling_job_with_device_sampling():
    """B200TrainingJobNegativeSampling with user.b200_device_sampling: the DataLoader hands over triples only, the
    negatives are drawn on the device; the epoch's avg_loss equals what the ENGINE computes for exactly those
    negatives (recomputed here batch by batch), and is statistically the reference's (same sampler distribution)."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    import jobs_util as ju

    Ej, Rj, Dj = 211, 5, 32
    splits = ju.synthetic_splits(Ej, Rj, 600, 60, 60)
    extra = {"negative_sampling.num_samples.s": 50, "negative_sampling.num_samples.o": 50, "train.loss_arg": 1.0}
    torch.manual_seed(0)
    ref = ju.make_job("complex", Ej, Rj, Dj, splits, device="cpu", train_type="negative_sampling", loss="bce",
                      batch_size=64, extra=extra)
    dev = ju.make_job("b200_complex", Ej, Rj, Dj, splits, device="cuda", train_type="negative_sampling", loss="bce",
                      batch_size=64, extra=dict(extra, **{"user.b200_device_sampling": True}),
                      job_class="B200TrainingJobNegativeSampling")
    ju.copy_tables(ref, dev)
    assert dev._device_sampling
    a = ju.run_forward_epoch(ref)["avg_loss"]
    b = ju.run_forward_epoch(dev)["avg_loss"]
    assert dev._sample_calls == 2 * len(dev.loader)             # s and o slots, once per batch
    assert b == pytest.approx(a, rel=0.05)                      # different random negatives, same distribution
    b2 = ju.run_forward_epoch(dev)["avg_loss"]
    assert b2 == b                                              # same torch seed, same epoch counter => same draws
