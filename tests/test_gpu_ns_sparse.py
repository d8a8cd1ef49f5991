"""Row-sparse table gradients of the negative-sampling step on the H100 (b200kge_ns_backward_sparse): the rows equal the
mirror's row set exactly; the values, scattered to dense, meet 1e-4 of the fp64 oracle's rms and agree with
b200kge_ns_backward's dense gradient, which is exactly 0 outside the set; and the job with `sparse: True` trains like
the reference job with Adagrad and SparseAdam."""
import pytest
import torch

import ns_dropout_oracle as nso
import ns_loss_oracle as nlo
import ns_sparse_oracle as nsp
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4
S, O = 0, 2
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]
LOSSES = {"bce": 0.25, "kl": 0.0, "margin_ranking": 1.0}


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


def _close(got, ref, what, tol=TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = float((got - ref).abs().max())
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


def _problem(model, E, R, D, n, K, seed):
    d = min(D, 16) if model == "rescal" else D
    ent, rel = orc.make_tables(model, E, R, d, sigma=0.5, seed=seed)
    tri = orc.make_triples(E, R, n, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    neg = torch.randint(0, E, (n, K), generator=g)
    if K > 4:
        neg[:, 3] = neg[:, 4]                 # repeats within a row
    return ent, rel, tri, neg


def _run(eng, model, ln, slot, loss, impl, drop, E, R, D, n, K, seed=0, oracle=True):
    ent, rel, tri, neg = _problem(model, E, R, D, n, K, seed)
    ec, rc, tc, nc = ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda()
    arg, bs = LOSSES[loss], n + 3
    key = eng.DropoutKey(0.3, 0.2, 99, 7, 5) if drop else None
    kw = {} if key is None else {"dropout": key, "implementation": impl}
    G = None
    if drop or loss != "bce":
        z = eng.ns_score(model, ec, rc, tc, nc, slot, True, ln, **kw)
        G = eng.ns_loss(z, loss, arg, 1.0, batch_size=bs, want_grad=True)[1]
    d_ent, d_rel = eng.ns_backward_sparse(model, ec, rc, tc, slot, nc, arg, ln, bs, grad_scores=G, **kw)
    assert d_ent.is_sparse and d_rel.is_sparse and d_ent.is_coalesced()
    want_e, want_r = nsp.row_sets(tri.numpy(), neg.numpy(), impl, E)
    assert torch.equal(d_ent.indices()[0].cpu(), torch.from_numpy(want_e))
    assert torch.equal(d_rel.indices()[0].cpu(), torch.from_numpy(want_r))
    dense_e, dense_r = d_ent.to_dense(), d_rel.to_dense()
    # the dense entry under the same operands: same atomics, so the same sums up to their order; 0 off the set
    ref_e, ref_r = eng.ns_backward(model, ec, rc, tc, {slot: nc}, arg, ln, bs,
                                   grad_scores=None if G is None else {slot: G}, **kw)
    off = torch.ones(E, dtype=torch.bool)
    off[torch.from_numpy(want_e)] = False
    assert not ref_e.cpu()[off].any()
    _close(dense_e, ref_e, "d_ent vs dense entry")
    _close(dense_r, ref_r, "d_rel vs dense entry")
    if not oracle:
        return
    if drop:
        e64, r64 = ent.double().requires_grad_(True), rel.double().requires_grad_(True)
        z64 = nso.block(model, e64, r64, tri, slot, neg, key, impl, ln)
        (z64 * G.double().cpu()).sum().backward()
        o_e, o_r = e64.grad, r64.grad
    else:
        o_e, o_r = nlo.ns_backward(model, ent.double(), rel.double(), tri, {slot: neg}, loss, arg, 1.0, ln, bs)
    _close(dense_e, o_e, f"{model} {loss} d_ent vs fp64")
    _close(dense_r, o_r, f"{model} {loss} d_rel vs fp64")


@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("loss", list(LOSSES))
@pytest.mark.parametrize("slot", [S, O])
@pytest.mark.parametrize("model,ln", CASES)
def test_rows_and_values_small(eng, model, ln, slot, loss, impl, drop):
    _run(eng, model, ln, slot, loss, impl, drop, 50, 6, 16, 3, 7)


@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("model,ln", [("complex", 1.0), ("transe", 2.0), ("rotate", 1.0)])
def test_rows_and_values_fb15k_shape(eng, model, ln, drop):
    _run(eng, model, ln, O, "kl", "batch", drop, 40943, 11, 128, 512, 1000, seed=3)


def test_all_gives_every_entity_row(eng):
    _run(eng, "complex", 1.0, S, "kl", "all", True, 300, 6, 16, 5, 20, oracle=False)


def test_row_map_at_wikidata5m_scale(eng):
    """E = 4.8M rows: the map, the tile scan (1172 tiles) and the compaction at scale; no fp64 oracle at this size."""
    _run(eng, "distmult", 1.0, O, "kl", "batch", False, 4_800_000, 20, 64, 512, 1000, seed=5, oracle=False)


def test_mixed_layout(eng):
    """A sparse entity table with a dense relation table, and the other way round."""
    ent, rel, tri, neg = _problem("complex", 200, 6, 16, 9, 11, 2)
    ec, rc, tc, nc = ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda()
    ref_e, ref_r = eng.ns_backward("complex", ec, rc, tc, {O: nc}, 0.5, 1.0, 20)
    for sp in ((True, False), (False, True)):
        d_e, d_r = eng.ns_backward_sparse("complex", ec, rc, tc, O, nc, 0.5, 1.0, 20, sparse=sp)
        assert d_e.is_sparse == sp[0] and d_r.is_sparse == sp[1]
        _close(d_e.to_dense() if d_e.is_sparse else d_e, ref_e, "d_ent")
        _close(d_r.to_dense() if d_r.is_sparse else d_r, ref_r, "d_rel")


# ---- the job: two epochs with `sparse: True` on both tables against the reference job fed the same negatives
from kge_b200 import hostenv  # noqa: E402

E_J, R_J, D_J = 60, 5, 16


def _job_pair(extra, model="complex"):
    import jobs_util as ju

    splits = ju.synthetic_splits(E_J, R_J, 150, 20, 20)
    torch.manual_seed(0)
    extra = dict(extra)
    extra.update({"lookup_embedder.sparse": True, "negative_sampling.num_samples.s": 5,
                  "negative_sampling.num_samples.o": 6, "train.loss_arg": 1.0})
    init = ju.make_job(model, E_J, R_J, D_J, splits, train_type="negative_sampling", loss="kl", batch_size=16,
                       extra=extra)
    jobs = {}
    for tag in ("ref", "plugin"):
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "plugin" else {}
        name, dev = (model, "cpu") if tag == "ref" else ("b200_" + model, "cuda")
        jobs[tag] = ju.make_job(name, E_J, R_J, D_J, splits, device=dev, train_type="negative_sampling", loss="kl",
                                batch_size=16, forward_only=False, extra=extra, **kw)
        ju.copy_tables(init, jobs[tag])
    return jobs


def _record_layouts(job):
    """The layout of every parameter's .grad at each optimizer step (before the step and its zero_grad)."""
    seen = []
    step = job.optimizer.step

    def recording_step(*a, **kw):
        seen.append(tuple(p.grad is not None and p.grad.is_sparse for p in job.model.parameters()))
        return step(*a, **kw)
    job.optimizer.step = recording_step
    return seen


needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")


@needs_ref
@pytest.mark.parametrize("optimizer", ["Adagrad", "SparseAdam"])
@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
def test_job_sparse_matches_reference(eng, optimizer, impl):
    import jobs_util as ju

    jobs = _job_pair({"train.optimizer.default.type": optimizer, "negative_sampling.implementation": impl})
    seen = _record_layouts(jobs["plugin"])
    for ep in range(2):
        losses = {}
        for tag, job in jobs.items():
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses[tag] = job.run_epoch()["avg_loss"]
        assert losses["plugin"] == pytest.approx(losses["ref"], rel=1e-4), (ep, losses)
    w_ref = jobs["ref"].model.get_s_embedder()._embeddings.weight.detach()
    w_plg = jobs["plugin"].model.get_s_embedder()._embeddings.weight.detach().cpu()
    _close(w_plg, w_ref, "trained entity table", tol=1e-4)
    assert seen and all(all(layout) for layout in seen), seen


# device sampling (frequency, filtered), the reciprocal wrapper, `user.b200_ns_dropout` and Lp penalties, each with
# `sparse: True` on both tables: the reference job replays the device's draws (and, with dropout, the mirror's masks)
JE, JR, JD = 211, 5, 32
P_ENT, P_REL = 0.3, 0.1


@pytest.fixture(scope="module")
def dev_splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _device_pair(splits, optimizer, recip, dropout, penalty, monkeypatch):
    import jobs_util as ju
    from kge_b200 import engine

    cfg = {"negative_sampling.implementation": "triple", "negative_sampling.num_samples.s": 7,
           "negative_sampling.num_samples.o": 9, "negative_sampling.filtering.s": True,
           "negative_sampling.filtering.o": True, "train.optimizer.default.type": optimizer,
           "lookup_embedder.sparse": True}
    if penalty:
        cfg.update({"lookup_embedder.regularize": "lp", "lookup_embedder.regularize_weight": 1e-2,
                    "lookup_embedder.regularize_args.weighted": penalty == "weighted"})
    drawn = {S: [], O: []}
    for name in ("sample_frequency", "sample_frequency_filtered"):
        orig = getattr(engine, name)

        def spy(*a, orig=orig, name=name, **kw):
            out = orig(*a, **kw)
            drawn[a[6] if name == "sample_frequency_filtered" else (a[4] & 3)].append(out.cpu())
            return out
        monkeypatch.setattr(engine, name, spy)

    def make(tag, dev):
        m = "complex" if tag == "ref" else "b200_complex"
        c, imports, model = dict(cfg), (), m
        if recip:
            c["reciprocal_relations_model.base_model.type"] = m
            model, imports = "reciprocal_relations_model", (m,)
        if dropout:
            c.update({f"{m}.entity_embedder.dropout": P_ENT, f"{m}.relation_embedder.dropout": P_REL})
        if tag == "b200":
            c.update({"user.b200_device_sampling": True, "negative_sampling.sampling_type": "frequency"})
            if dropout:
                c["user.b200_ns_dropout"] = True
        return ju.make_job(model, JE, JR, JD, splits, device=dev, train_type="negative_sampling", loss="kl",
                           batch_size=64, forward_only=False, extra=c, imports=imports,
                           job_class="B200TrainingJobNegativeSampling" if tag == "b200" else None)

    torch.manual_seed(0)
    init = make("ref", "cpu")
    out = {}
    for tag in ("b200", "ref"):
        job = make(tag, "cuda")
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        if tag == "b200":
            assert job._device_sampling and sorted(job._frequency) == [S, O] and sorted(job._filter_index) == [S, O]
            seen = _record_layouts(job)
        else:
            if dropout:
                nso.patch_reference_ns_job(job, P_ENT, P_REL)
            queue = {slot: list(v) for slot, v in drawn.items()}
            job._sampler._sample = lambda tri, slot, num: (queue[slot].pop(0)[: len(tri), :num].clone() if num > 0
                                                           else torch.empty((len(tri), 0), dtype=torch.int64))
            seen = _record_layouts(job)
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        if tag == "ref":
            assert not any(queue.values())
        out[tag] = (losses, [p.detach().cpu() for p in job.model.parameters()], seen)
    return out


@needs_ref
@pytest.mark.parametrize("optimizer", ["Adagrad", "SparseAdam"])
@pytest.mark.parametrize("recip,dropout,penalty", [(False, False, None), (True, False, None), (False, True, None),
                                                   (False, False, "weighted"), (False, False, "unweighted"),
                                                   (True, False, "weighted")])
def test_device_sampling_job_sparse_matches_reference(eng, dev_splits, optimizer, recip, dropout, penalty,
                                                      monkeypatch):
    out = _device_pair(dev_splits, optimizer, recip, dropout, penalty, monkeypatch)
    assert out["b200"][0][0] == pytest.approx(out["ref"][0][0], rel=TOL)
    assert out["b200"][0][1] == pytest.approx(out["ref"][0][1], rel=1e-3)
    for k, (a, b) in enumerate(zip(out["b200"][1], out["ref"][1])):
        _close(a, b, f"parameter {k}", 10 * TOL)
    # every step saw row-sparse gradients on both tables, in the reference job and in the plugin's
    for tag in ("b200", "ref"):
        assert out[tag][2] and all(all(layout) for layout in out[tag][2]), (tag, out[tag][2][:3])


@pytest.mark.parametrize("weighted", [True, False])
def test_penalty_gradient_of_a_sparse_embedder(eng, weighted):
    """The patched penalty of a `sparse: True` embedder: weighted, row-sparse over unique(indexes); unweighted, over
    every row (the reference's embed_all()); the values are the dense autograd gradient of the reference expression."""
    import jobs_util as ju

    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    cfg = {"lookup_embedder.sparse": True, "lookup_embedder.regularize": "lp", "lookup_embedder.regularize_weight": 0.3,
           "lookup_embedder.regularize_args.weighted": weighted, "lookup_embedder.regularize_args.p": 3}
    job = ju.make_job("b200_complex", JE, JR, JD, ju.synthetic_splits(JE, JR, 60), device="cuda",
                      train_type="negative_sampling", loss="kl", batch_size=16, forward_only=False, extra=cfg,
                      job_class="B200TrainingJobNegativeSampling")
    from kge_b200.plugin import _penalty_torch         # after make_job: the plugin imports the reference

    emb = job.model.get_s_embedder()
    w = emb._embeddings.weight
    idx = torch.tensor([5, 3, 5, 200, 3, 3, 17], device="cuda")
    (val,) = [v for k, v in emb.penalty(indexes=idx) if k.endswith("_penalty")]
    (2.5 * val).backward()
    assert w.grad.is_sparse
    want_rows = torch.unique(idx) if weighted else torch.arange(JE, device="cuda")
    assert w.grad._nnz() == len(want_rows)            # one entry per row: nothing for coalesce() to merge
    grad = w.grad.coalesce()
    assert torch.equal(grad.indices()[0], want_rows)
    wd = w.detach().clone().requires_grad_(True)
    (dense,) = torch.autograd.grad(2.5 * _penalty_torch(emb, wd, "lp", 0.3, 3, weighted, idx if weighted else None),
                                   wd)
    _close(grad.values(), dense[want_rows], "penalty gradient rows")
