"""The negative-sampling P slot on the H100 (b200kge_ns_p_backward): table gradients against fp64 autograd of the
reference's block (oracle.ns_scores_with_positive, slot P) under each loss's fp64 gradient, within 1e-4 of the fp64 rms
per table; the row-sparse layout's rows equal the rows the reference looks up and its values the dense entry's; and the
job with `user.b200_ns_p_slot: true` trains like the unmodified reference job fed the same negatives."""
import pytest
import torch

import ns_loss_oracle as nlo
from kge_b200 import hostenv
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4
S, P, O = 0, 1, 2
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]
LOSSES = {"bce": 0.25, "kl": 0.0, "margin_ranking": 1.0, "bce_self_adversarial": 0.5}


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


def _close(got, ref, what, tol=TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = float((got - ref).abs().max())
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-12)
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


def _problem(model, E, R, D, n, K, seed):
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5, seed=seed)
    tri = orc.make_triples(E, R, n, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    neg = torch.randint(0, R, (n, K), generator=g)
    if K > 4:
        neg[:, 3] = neg[:, 4]                 # repeats within a row
        neg[:, 0] = tri[:, 1]                 # the positive's own relation drawn as a negative
    return ent, rel, tri, neg


def _reference_rows(tri, neg, impl, R):
    """The rows the reference looks up for a P slot: s and o; p and every sampled id (every relation for "all")."""
    ent_rows = torch.unique(torch.cat((tri[:, 0], tri[:, 2])))
    rel_rows = torch.arange(R) if impl == "all" else torch.unique(torch.cat((tri[:, 1], neg.reshape(-1))))
    return ent_rows, rel_rows


def _run(eng, model, ln, loss, impl, E, R, D, n, K, seed=0, sparse=False):
    ent, rel, tri, neg = _problem(model, E, R, D, n, K, seed)
    ec, rc, tc, nc = ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda()
    arg, bs = LOSSES[loss], n + 3
    z = eng.ns_score(model, ec, rc, tc, nc, P, True, ln)
    G = eng.ns_loss(z, loss, arg, 0.7, batch_size=bs, want_grad=True)[1]
    d_ent, d_rel = eng.ns_p_backward(model, ec, rc, tc, nc, G, ln, impl)
    # fp64: the reference's block under the loss's own gradient
    e64, r64 = ent.double().requires_grad_(True), rel.double().requires_grad_(True)
    z64 = orc.ns_scores_with_positive(model, e64, r64, tri, neg, P, impl, ln)
    G64 = nlo.ns_loss_grad(z64.detach(), loss, arg, 0.7, None, bs)
    (z64 * G64).sum().backward()
    _close(d_ent, e64.grad, f"{model} L{ln} {loss} {impl} d_ent")
    _close(d_rel, r64.grad, f"{model} L{ln} {loss} {impl} d_rel")
    if not sparse:
        return
    s_ent, s_rel = eng.ns_p_backward(model, ec, rc, tc, nc, G, ln, impl, sparse=(True, True))
    assert s_ent.is_sparse and s_rel.is_sparse and s_ent.is_coalesced() and s_rel.is_coalesced()
    want_e, want_r = _reference_rows(tri, neg, impl, R)
    assert torch.equal(s_ent.indices()[0].cpu(), want_e)
    assert torch.equal(s_rel.indices()[0].cpu(), want_r)
    # the dense entry under the same operands: the entity rows' atomics add in another order
    _close(s_ent.to_dense(), d_ent, "sparse d_ent vs dense entry")
    _close(s_rel.to_dense(), d_rel, "sparse d_rel vs dense entry")
    off = torch.ones(E, dtype=torch.bool)
    off[want_e] = False
    assert not d_ent.cpu()[off].any()


@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
@pytest.mark.parametrize("loss", list(LOSSES))
@pytest.mark.parametrize("model,ln", CASES)
def test_entry_small(eng, model, ln, loss, impl):
    _run(eng, model, ln, loss, impl, 50, 11, 16, 5, 7, sparse=True)


@pytest.mark.parametrize("K", [1, 1000])
@pytest.mark.parametrize("R", [11, 237])
@pytest.mark.parametrize("model,ln", CASES)
def test_entry_benchmark_shapes(eng, model, ln, R, K):
    D = 32 if model == "rescal" else 128
    _run(eng, model, ln, "kl", "batch", 2000, R, D, 512, K, seed=3, sparse=(K == 1000))


def test_entry_repeats_and_mixed_layouts(eng):
    """K > R forces every row to repeat relations; one table sparse, the other dense."""
    ent, rel, tri, neg = _problem("rotate", 300, 11, 32, 64, 40, 5)
    ec, rc, tc, nc = ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda()
    G = eng.ns_loss(eng.ns_score("rotate", ec, rc, tc, nc, P, True, 1.0), "kl", want_grad=True, batch_size=64)[1]
    ref_e, ref_r = eng.ns_p_backward("rotate", ec, rc, tc, nc, G, 1.0)
    for sp in ((True, False), (False, True)):
        d_e, d_r = eng.ns_p_backward("rotate", ec, rc, tc, nc, G, 1.0, sparse=sp)
        assert d_e.is_sparse == sp[0] and d_r.is_sparse == sp[1]
        _close(d_e.to_dense() if d_e.is_sparse else d_e, ref_e, "d_ent")
        _close(d_r.to_dense() if d_r.is_sparse else d_r, ref_r, "d_rel")


def test_rescal_above_d32_is_reported(eng):
    """RESCAL's [D, D] relation rows at D = 64: the measured error, held to 1e-4 of the fp64 rms as below D = 32."""
    _run(eng, "rescal", 1.0, "kl", "batch", 300, 11, 64, 64, 20, seed=7)


def test_unserved_norm_and_too_many_relations_are_refused(eng):
    ent, rel, tri, neg = _problem("transe", 50, 11, 16, 5, 7, 0)
    G = torch.zeros((5, 8), device="cuda")
    with pytest.raises(NotImplementedError):
        eng.ns_p_backward("transe", ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda(), G, 3.0)
    from kge_b200._lib import NS_P_MAX_RELATIONS

    big = torch.zeros((NS_P_MAX_RELATIONS + 1, 16), device="cuda")
    with pytest.raises(NotImplementedError):
        eng.ns_p_backward("distmult", ent.cuda(), big, tri.cuda(), neg.cuda(), G, 1.0)


# ---- the job: two epochs with the option on against the unmodified reference job fed the same negatives
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 211, 7, 32
SAMPLERS = ("sample_uniform", "sample_uniform_filtered", "sample_frequency", "sample_frequency_filtered")


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _train_pair(splits, model, optimizer, sparse, device, monkeypatch, loss="kl"):
    import jobs_util as ju
    from kge_b200 import engine

    cfg = {"negative_sampling.implementation": "triple", "negative_sampling.num_samples.s": 5,
           "negative_sampling.num_samples.p": 9, "negative_sampling.num_samples.o": 6,
           "train.optimizer.default.type": optimizer, "lookup_embedder.sparse": sparse, "train.loss_arg": 1.0}
    drawn = {S: [], P: [], O: []}
    for name in SAMPLERS:
        orig = getattr(engine, name)

        def spy(*a, orig=orig, **kw):
            out = orig(*a, **kw)
            drawn[a[4] & 3].append(out.cpu())          # offset = (epoch, batch) << 2 | slot
            return out
        monkeypatch.setattr(engine, name, spy)

    def make(tag):
        m = model if tag == "ref" else "b200_" + model
        c = dict(cfg)
        if tag == "b200":
            c["user.b200_ns_p_slot"] = True
            if device:
                c["user.b200_device_sampling"] = True
                if device == "filtered":
                    c["negative_sampling.filtering.p"] = True
                elif device == "frequency":
                    c["negative_sampling.sampling_type"] = "frequency"
        return ju.make_job(m, JE, JR, JD, splits, device="cuda" if tag == "b200" else "cpu",
                           train_type="negative_sampling", loss=loss, batch_size=64, forward_only=False, extra=c,
                           job_class="B200TrainingJobNegativeSampling" if tag == "b200" else None)

    torch.manual_seed(0)
    init = make("ref")
    out = {}
    for tag in ("b200", "ref"):
        job = make(tag)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        if tag == "ref" and device:
            queue = {slot: list(v) for slot, v in drawn.items()}
            job._sampler._sample = lambda tri, slot, num: queue[slot].pop(0)[: len(tri), :num].clone()
        calls = {"p": 0}
        if tag == "b200":
            orig_p = engine.ns_p_backward

            def counted(*a, **kw):
                calls["p"] += 1
                return orig_p(*a, **kw)
            monkeypatch.setattr(engine, "ns_p_backward", counted)
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        if tag == "b200":
            assert calls["p"] > 0 and job._device_sampling == bool(device)
        else:
            if device:
                assert not any(queue.values())
        out[tag] = (losses, [p.detach().cpu() for p in job.model.parameters()])
    return out


@needs_ref
@pytest.mark.parametrize("model,optimizer,sparse,device", [
    ("complex", "Adagrad", False, None), ("complex", "Adagrad", True, None), ("complex", "SparseAdam", True, None),
    ("rotate", "Adagrad", False, None), ("transe", "Adagrad", True, None),
    ("complex", "Adagrad", False, "uniform"), ("complex", "SparseAdam", True, "filtered"),
    ("distmult", "Adagrad", False, "frequency")])
def test_job_matches_the_reference_job(eng, splits, model, optimizer, sparse, device, monkeypatch):
    out = _train_pair(splits, model, optimizer, sparse, device, monkeypatch)
    assert out["b200"][0][0] == pytest.approx(out["ref"][0][0], rel=TOL)
    assert out["b200"][0][1] == pytest.approx(out["ref"][0][1], rel=1e-3)
    for k, (a, b) in enumerate(zip(out["b200"][1], out["ref"][1])):
        _close(a, b, f"parameter {k}", 10 * TOL)
