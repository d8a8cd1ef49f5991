"""Reciprocal-relations training on the H100: the reciprocal 1vsAll step (loss, d_ent, all 2R rows of d_rel) and the
KvsAll _po query type (sp_ fold of (o, p + R) on the _po mask streams) against fp64 autograd of the reference expression
(reciprocal_relations_model.py:85-92), with and without dropout, and two training epochs of each job plugin on a
ReciprocalRelationsModel against the unmodified wrapper job on the CPU."""
import pytest
import torch

import dropout_oracle as dro
import philox_np
from kge_b200 import hostenv
from test_gpu_dropout import _score      # RotatE L1 with the kernels' gradient at exact ties

pytestmark = pytest.mark.gpu

TOL = 1e-4          # of the reference gradient's rms (tests/test_gpu_backward.py)
TOL_ENT = 3e-4      # d_ent rows that sum thousands of fp32 terms (reasoning in tests/test_gpu_dropout_shapes.py)
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


@pytest.fixture()
def fast_mirror(monkeypatch):
    monkeypatch.setattr(dro, "mask", philox_np.mask)


def _close(got, ref, what, tol=TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = float((got - ref).abs().max())
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


def _tables(model, E, R, D, n, seed=0):
    from oracle import kge_oracle as orc

    g = torch.Generator().manual_seed(seed)
    ent = torch.randn(E, D, generator=g) * 0.3
    rel = torch.randn(2 * R, orc.relation_dim(model, D), generator=g) * 0.3
    tri = torch.stack([torch.randint(0, E, (n,), generator=g), torch.randint(0, R, (n,), generator=g),
                       torch.randint(0, E, (n,), generator=g)], 1)
    return ent, rel, tri


def _ref_recip(model, ent, rel, tri, R, loss, offset, key, l_norm):
    """(loss(score_sp(s, p), o) + loss(score_sp(o, p + R), s)) / n, the second direction on the _po draws."""
    from oracle import kge_oracle as orc

    s, p, o = tri[:, 0], tri[:, 1], tri[:, 2]
    total = 0.0
    for direction, a, pr, lab in ((0, s, p, o), (1, o, p + R, s)):
        q, r, t = ent[a], rel[pr], ent
        if key is not None:
            sq, sr, st = dro.DIR_STREAMS[direction]
            q = dro.apply(q, key.p_ent, key.seed, key.call, sq, key.row_base)
            r = dro.apply(r, key.p_rel, key.seed, key.call, sr, key.row_base)
            t = dro.apply(t, key.p_ent, key.seed, key.call, st, 0)
        x = _score(model, q, r, t, "sp_", l_norm)
        total = total + (orc.bce_loss(x, lab, offset) if loss == "bce" else orc.kl_loss(x, lab))
    return total / tri.shape[0]


def _check_recip(eng, model, l_norm, loss, E, R, D, n, key, tol_ent=TOL):
    ent, rel, tri = _tables(model, E, R, D, n)
    offset = 0.5 if loss == "bce" else 0.0
    val, de, dr = dro.grads(lambda e, r: _ref_recip(model, e, r, tri, R, loss, offset, key, l_norm),
                            ent.double(), rel.double())
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    got = eng.train_1vsall_reciprocal_forward(model, ec, rc, tc, R, loss, offset, l_norm, dropout=key)
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.train_1vsall_reciprocal_backward(model, ec, rc, tc, R, loss, offset, l_norm, dropout=key)
    assert gr.shape[0] == 2 * R
    _close(ge, de, "d_ent", tol_ent)
    _close(gr, dr, "d_rel")


@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,l_norm", CASES)
def test_reciprocal_1vsall_toy(eng, model, l_norm, loss, drop):
    key = eng.DropoutKey(0.3, 0.2, seed=2024, call=77, row_base=130) if drop else None
    _check_recip(eng, model, l_norm, loss, 300, 7, 32, 64, key)


@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("model,l_norm", [("complex", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 2.0),
                                          ("rotate", 1.0)])
def test_reciprocal_1vsall_multi_tile(eng, fast_mirror, model, l_norm, drop):
    """E=5003, n=600: split-K backward GEMMs, several scorer tiles, CP (K=128) on the tensor cores."""
    key = eng.DropoutKey(0.4, 0.2, seed=5, call=9, row_base=600) if drop else None
    D = 64 if model == "rescal" else 256
    _check_recip(eng, model, l_norm, "kl", 5003, 11, D, 600, key, TOL_ENT)


@pytest.mark.parametrize("drop", [False, True])
def test_reciprocal_1vsall_bench_shape(eng, fast_mirror, drop):
    key = eng.DropoutKey(0.4, 0.2, seed=1, call=2, row_base=0) if drop else None
    _check_recip(eng, "complex", 1.0, "bce", 14541, 237, 512, 1024, key, TOL_ENT)


def test_reciprocal_refuses_wrong_relation_count(eng):
    ent, rel, tri = _tables("complex", 50, 4, 16, 8)
    with pytest.raises(ValueError):
        eng.train_1vsall_reciprocal_forward("complex", ent.cuda(), rel.cuda(), tri.cuda(), 5)


def _csr(n, E, seed=1):
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(1, 5, (n,), generator=g)
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(counts, 0)
    cols = torch.cat([torch.sort(torch.randint(0, E, (int(c),), generator=g))[0] for c in counts])
    return offs, cols


@pytest.mark.parametrize("eps", [0.0, 0.2])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model", ["complex", "distmult", "simple", "cp", "rescal"])
def test_kvsall_reciprocal_po_with_dropout(eng, model, loss, eps):
    """A reciprocal _po query type: sp_ fold of (o, p + R), labels over subjects, masks on the _po streams."""
    from oracle import kge_oracle as orc

    E, R, D, n = 300, 7, 32, 64
    ent, rel, tri = _tables(model, E, R, D, n, seed=3)
    o, pr = tri[:, 2], tri[:, 1] + R
    offs, cols = _csr(n, E)
    key = eng.DropoutKey(0.3, 0.2, seed=99, call=5, row_base=40)
    offset = 0.5 if loss == "bce" else 0.0
    bs = 2 * n

    def ref(e, r):
        sq, sr, st = dro.DIR_STREAMS[1]
        q = dro.apply(e[o], key.p_ent, key.seed, key.call, sq, key.row_base)
        rr = dro.apply(r[pr], key.p_rel, key.seed, key.call, sr, key.row_base)
        t = dro.apply(e, key.p_ent, key.seed, key.call, st, 0)
        x = orc.score_emb(model, q, rr, t, "sp_", 1.0)
        y = torch.zeros(x.shape, dtype=x.dtype)
        rows = torch.repeat_interleave(torch.arange(n), offs[1:] - offs[:-1])
        y.index_put_((rows, cols), torch.ones(len(rows), dtype=x.dtype), accumulate=True)
        if eps > 0:
            y = orc.kvsall_smooth_labels(y, eps)
        return (orc.bce_loss(x, y, offset) if loss == "bce" else orc.kl_loss(x, y)) / bs

    val, de, dr = dro.grads(ref, ent.double(), rel.double())
    ec, rc = ent.cuda(), rel.cuda()
    qc, pc, oc, cc = o.cuda(), pr.cuda(), offs.cuda(), cols.cuda()
    got = eng.score_1vsN_loss_csr(model, "sp_", ec, rc, ec, oc, cc, qc, pc, loss, offset, eps, dropout=key,
                                  dropout_streams="_po") / bs
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.score_1vsN_loss_csr_backward(model, "sp_", ec, rc, qc, pc, oc, cc, loss, offset, eps, bs, dropout=key,
                                              dropout_streams="_po")
    _close(ge, de, "d_ent")
    _close(gr, dr, "d_rel")


# ---- job plugins on the wrapper against the unmodified wrapper job -------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 211, 5, 32
REL = 1e-4


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _run_pair(base, train_type, loss, job_class, extra, splits, device_sampling=False, dropout=False):
    import jobs_util as ju

    hostenv.import_kge()
    from kge.model.embedder.lookup_embedder import LookupEmbedder

    def make(bm, dev, cls):
        cfg = {"reciprocal_relations_model.base_model.type": bm}
        cfg.update(extra)
        if dropout:
            cfg.update({f"{bm}.entity_embedder.dropout": 0.3, f"{bm}.relation_embedder.dropout": 0.1})
        if cls and device_sampling:
            cfg["user.b200_device_sampling"] = True
        return ju.make_job("reciprocal_relations_model", JE, JR, JD, splits, device=dev, train_type=train_type,
                           loss=loss, batch_size=64, forward_only=False, imports=(bm,), extra=cfg, job_class=cls)

    torch.manual_seed(0)
    init = make(base, "cpu", None)
    out = {}
    for tag, dev, bm, cls in (("ref", "cpu", base, None), ("b200", "cuda", "b200_" + base, job_class)):
        job = make(bm, dev, cls)
        if tag == "ref" and dropout:
            dro.patch_reference_job(job, 0.3, 0.1)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        embed_all_calls = []
        if tag == "b200":
            orig = LookupEmbedder.embed_all
            for emb in (job.model.get_s_embedder(), job.model.get_p_embedder()):
                emb.embed_all = lambda emb=emb: embed_all_calls.append(1) or orig(emb)
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(20 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        out[tag] = losses
        if tag == "b200":
            assert not embed_all_calls                  # the native route ran, not the reference step
    return out


def _assert_tracks(out, rel1=REL):
    assert out["b200"][0] == pytest.approx(out["ref"][0], rel=rel1)
    assert out["b200"][1] == pytest.approx(out["ref"][1], rel=1e-3)


@needs_ref
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("base,loss", [("complex", "kl"), ("rescal", "bce"), ("cp", "kl"), ("transe", "kl"),
                                       ("rotate", "bce")])
def test_1vsall_job_on_wrapper(eng, base, loss, dropout, splits):
    _assert_tracks(_run_pair(base, "1vsAll", loss, "B200TrainingJob1vsAll", {}, splits, dropout=dropout))


@needs_ref
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("base,loss,eps", [("complex", "kl", 0.0), ("distmult", "bce", 0.1)])
def test_kvsall_job_on_wrapper(eng, base, loss, eps, dropout, splits):
    _assert_tracks(_run_pair(base, "KvsAll", loss, "B200TrainingJobKvsAll", {"KvsAll.label_smoothing": eps}, splits,
                             dropout=dropout))


@needs_ref
@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("base", ["complex", "transe"])
def test_negative_sampling_job_on_wrapper(eng, base, impl, splits):
    extra = {"negative_sampling.implementation": impl, "negative_sampling.num_samples.s": 7,
             "negative_sampling.num_samples.o": 9, "train.loss_arg": 2.0}
    _assert_tracks(_run_pair(base, "negative_sampling", "kl", "B200TrainingJobNegativeSampling", extra, splits))


@needs_ref
@pytest.mark.parametrize("base", ["complex", "transe"])
def test_negative_sampling_device_sampling_on_wrapper(eng, base, splits):
    """Device-drawn negatives (the reference cannot consume them): every checked sub-batch's S- and O-slot loss equals
    the kl of the wrapper's own reference scores of the same negatives (S slot: score_spo(o, p + R, s'))."""
    import jobs_util as ju

    hostenv.import_kge()
    from kge_b200.plugin import _B200ScorerMixin

    extra = {"reciprocal_relations_model.base_model.type": "b200_" + base, "user.b200_device_sampling": True,
             "negative_sampling.num_samples.s": 5, "negative_sampling.num_samples.o": 6}
    job = ju.make_job("reciprocal_relations_model", JE, JR, JD, splits, device="cuda", train_type="negative_sampling",
                      loss="kl", batch_size=64, forward_only=False, imports=("b200_" + base,), extra=extra,
                      job_class="B200TrainingJobNegativeSampling")
    model = job.model
    base_model = model._base_model
    checked = []
    orig = base_model.loss_negatives

    def loss_negatives(tri, neg, slot, offset, batch_size, loss="bce", temperature=1.0, **kw):
        val = orig(tri, neg, slot, offset, batch_size, loss, temperature, **kw)
        if len(checked) < 6:
            with torch.no_grad():
                e, r = (t.detach().double() for t in base_model._b200_weights())
                ref = super(_B200ScorerMixin, base_model._scorer).score_emb     # the reference expression
                cand = torch.cat((tri[:, 2:3], neg), 1)
                x = ref(e[tri[:, 0]].repeat_interleave(cand.shape[1], 0), r[tri[:, 1]].repeat_interleave(cand.shape[1], 0),
                        e[cand.reshape(-1)], "spo").view(len(tri), -1)
                want = -torch.log_softmax(x, 1)[:, 0].sum() / batch_size
            checked.append((slot, float(val), float(want)))
        return val
    base_model.loss_negatives = loss_negatives
    job.epoch += 1
    job._prepare()
    ju.seed_all(3)
    job.run_epoch()
    assert checked
    for slot, got, want in checked:
        assert got == pytest.approx(want, rel=1e-4), slot


@needs_ref
def test_reciprocal_p_slot_and_ns_dropout_keep_todays_route(eng, splits):
    import jobs_util as ju

    hostenv.import_kge()
    base = "b200_complex"
    for extra in ({"negative_sampling.num_samples.p": 3},
                  {f"{base}.entity_embedder.dropout": 0.3, "user.b200_ns_dropout": True}):
        cfg = {"reciprocal_relations_model.base_model.type": base, "user.b200_device_sampling": True}
        cfg.update(extra)
        job = ju.make_job("reciprocal_relations_model", JE, JR, JD, splits, device="cuda",
                          train_type="negative_sampling", loss="kl", batch_size=64, forward_only=False,
                          imports=(base,), extra=cfg, job_class="B200TrainingJobNegativeSampling")
        job.epoch += 1
        job._prepare()
        with pytest.raises(NotImplementedError, match="reciprocal_relations_model"):
            job.run_epoch()
