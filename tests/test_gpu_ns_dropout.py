"""Embedding dropout of the negative-sampling step on the H100: the mask kernel on the NS streams against the CPU mirror
bit for bit, b200kge_ns_score_dropout / b200kge_ns_backward (dropout key) against the fp64 masked expression of
tests/ns_dropout_oracle.py (and its autograd), determinism, and the job plugin with `user.b200_ns_dropout` against the
reference job drawing the mirror's masks."""
import pytest
import torch

import dropout_oracle as dro
import ns_dropout_oracle as nso
from kge_b200 import hostenv

pytestmark = pytest.mark.gpu

TOL = 1e-4          # of the reference's rms, as tests/test_gpu_dropout.py


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


@pytest.mark.parametrize("slot,j,rows,dim,row_base", [(0, 0, 5, 16, 3), (0, 4, 40, 16, 120), (2, 5, 9, 64, 0),
                                                      (2, 1, 3, 256, 7)])
def test_mask_kernel_matches_mirror_on_ns_streams(eng, slot, j, rows, dim, row_base):
    st = nso.stream(slot, j)
    got = eng.dropout_mask(0.3, 2 ** 35 + 11, 77, st, rows, dim, row_base).cpu().bool()
    assert torch.equal(got, dro.mask(0.3, 2 ** 35 + 11, 77, st, rows, dim, row_base))


E, R, D, N, K = 40, 5, 16, 6, 37
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]


def _problem(model, seed=0):
    g = torch.Generator().manual_seed(seed)
    d = 8 if model == "rescal" else D
    dr = {"rescal": d * d, "cp": d // 2, "rotate": d // 2}.get(model, d)
    ent = torch.randn(E, d, generator=g, dtype=torch.float64) * 0.5
    rel = torch.randn(R, dr, generator=g, dtype=torch.float64) * 0.5
    tri = torch.stack([torch.randint(0, E, (N,), generator=g), torch.randint(0, R, (N,), generator=g),
                       torch.randint(0, E, (N,), generator=g)], 1)
    neg = torch.randint(0, E, (N, K), generator=g)        # E < N K: ids repeat within and across rows
    neg[:, 3] = neg[:, 4]
    return ent, rel, tri, neg


def _key(eng, call=5, row_base=11):
    return eng.DropoutKey(0.3, 0.2, 1234567, call, row_base)


@pytest.mark.parametrize("model,l_norm", CASES)
@pytest.mark.parametrize("slot", [0, 2])
@pytest.mark.parametrize("impl", ["triple", "batch"])
def test_score_against_fp64(eng, model, l_norm, slot, impl):
    ent, rel, tri, neg = _problem(model)
    neg[:, 0] = tri[:, slot]                              # a negative equal to the positive entity
    key = _key(eng)
    got = eng.ns_score(model, ent.float().cuda(), rel.float().cuda(), tri.cuda(), neg.cuda(), slot, True, l_norm,
                       dropout=key, implementation=impl)
    ref = nso.block(model, ent, rel, tri, slot, neg, key, impl, l_norm)
    _close(got, ref, f"{model} slot {slot} {impl}")


@pytest.mark.parametrize("model,l_norm", CASES)
@pytest.mark.parametrize("slot", [0, 2])
@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("loss", ["kl", "bce", "margin_ranking", "bce_self_adversarial"])
def test_backward_against_fp64_autograd(eng, model, l_norm, slot, impl, loss):
    ent, rel, tri, neg = _problem(model, seed=1)
    key = _key(eng, call=9, row_base=3)
    e32, r32 = ent.float().cuda(), rel.float().cuda()
    scores = eng.ns_score(model, e32, r32, tri.cuda(), neg.cuda(), slot, True, l_norm, dropout=key, implementation=impl)
    _, G = eng.ns_loss(scores, loss, 1.0 if loss == "margin_ranking" else 0.0, 0.5, batch_size=N, want_grad=True)
    d_ent, d_rel = eng.ns_backward(model, e32, r32, tri.cuda(), {slot: neg.cuda()}, l_norm=l_norm,
                                   grad_scores={slot: G}, dropout=key, implementation=impl)
    _, de, dr = dro.grads(lambda e, r: (G.double().cpu() * nso.block(model, e, r, tri, slot, neg, key, impl,
                                                                          l_norm)).sum(), ent, rel)
    _close(d_ent, de, f"{model} d_ent")
    _close(d_rel, dr, f"{model} d_rel")


def test_same_key_is_deterministic_and_call_changes_masks(eng):
    ent, rel, tri, neg = _problem("complex")
    args = ("complex", ent.float().cuda(), rel.float().cuda(), tri.cuda(), neg.cuda(), 2, True, 1.0)
    for impl in ("triple", "batch"):
        a = eng.ns_score(*args, dropout=_key(eng), implementation=impl)
        b = eng.ns_score(*args, dropout=_key(eng), implementation=impl)
        c = eng.ns_score(*args, dropout=_key(eng, call=6), implementation=impl)
        assert torch.equal(a, b)
        assert not torch.equal(a, c)


def test_unsupported_configurations_are_refused(eng):
    ent, rel, tri, neg = _problem("complex")
    with pytest.raises(NotImplementedError):           # P slot
        eng.ns_score("complex", ent.float().cuda(), rel.float().cuda(), tri.cuda(), neg.cuda() % R, 1, True,
                     dropout=_key(eng))
    ent, rel, tri, neg = _problem("transe")
    with pytest.raises(NotImplementedError):           # TransE l_norm 3
        eng.ns_score("transe", ent.float().cuda(), rel.float().cuda(), tri.cuda(), neg.cuda(), 0, True, 3.0,
                     dropout=_key(eng))


# ---- the job plugin ------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 53, 4, 16
P_ENT, P_REL = 0.3, 0.1


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 150, 20, 20)


def _train_pair(model, splits, impl, Kn, loss="kl", subbatch=None, extra=None, l_norm=None):
    import jobs_util as ju

    # plain SGD, as tests/test_ns_dropout_cpu.py: Adagrad's first step turns fp32 rounding differences on near-zero
    # gradient elements into full-size steps
    cfg = {"negative_sampling.implementation": impl,
           "negative_sampling.num_samples.s": Kn, "negative_sampling.num_samples.o": Kn,
           "train.optimizer.default.type": "SGD", "train.optimizer.default.args.lr": 0.1}
    cfg.update(extra or {})
    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, train_type="negative_sampling", loss=loss, batch_size=32,
                       extra={**cfg, **({f"{model}.l_norm": l_norm} if l_norm is not None else {})})
    out = {}
    for name in ("ref", "plugin"):
        m = model if name == "ref" else "b200_" + model
        c = {f"{m}.entity_embedder.dropout": P_ENT, f"{m}.relation_embedder.dropout": P_REL, **cfg}
        if name == "plugin":
            c["user.b200_ns_dropout"] = True
        if l_norm is not None:
            c[f"{m}.l_norm"] = l_norm
        job = ju.make_job(m, JE, JR, JD, splits, device="cuda", train_type="negative_sampling", loss=loss,
                          batch_size=32, forward_only=False, extra=c,
                          job_class="B200TrainingJobNegativeSampling" if name == "plugin" else None)
        if name == "ref":
            nso.patch_reference_ns_job(job, P_ENT, P_REL)
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
        out[name] = (losses, job.model.get_s_embedder()._embeddings.weight.detach().cpu(),
                     job.model.get_p_embedder()._embeddings.weight.detach().cpu())
    return out


@needs_ref
@pytest.mark.parametrize("model,impl,Kn,subbatch,l_norm,loss", [
    ("complex", "triple", 3, None, None, "kl"), ("complex", "batch", 40, 12, None, "kl"),
    ("rotate", "triple", 3, None, None, "bce_self_adversarial"), ("rotate", "batch", 40, None, None, "kl"),
    ("transe", "triple", 3, None, 2.0, "margin_ranking"), ("transe", "batch", 40, None, 2.0, "kl"),
    ("rescal", "triple", 3, None, None, "kl"), ("rescal", "batch", 40, None, None, "bce")])
def test_job_with_ns_dropout_matches_the_reference(model, impl, Kn, subbatch, l_norm, loss, splits):
    out = _train_pair(model, splits, impl, Kn, loss=loss, subbatch=subbatch, l_norm=l_norm)
    assert out["plugin"][0] == pytest.approx(out["ref"][0], rel=TOL)
    for k in (1, 2):
        _close(out["plugin"][k], out["ref"][k], f"table {k}", tol=10 * TOL)


@needs_ref
def test_job_with_ns_dropout_and_device_sampling_trains(splits):
    """Device-drawn negatives with the dropout route: every sub-batch's loss equals the fp64 masked expression of the
    negatives and key it received."""
    import math

    import jobs_util as ju
    import ns_loss_oracle as nlo

    cfg = {"b200_complex.entity_embedder.dropout": P_ENT, "negative_sampling.implementation": "triple",
           "negative_sampling.num_samples.s": 3, "negative_sampling.num_samples.o": 3,
           "user.b200_ns_dropout": True, "user.b200_device_sampling": True}
    job = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", train_type="negative_sampling", loss="kl",
                      batch_size=32, forward_only=False, extra=cfg, job_class="B200TrainingJobNegativeSampling")
    checked = []
    orig = job.model.loss_negatives

    def spy(triples, negatives, slot, offset, batch_size, loss, temperature, dropout=None, implementation="batch"):
        assert dropout is not None and negatives.is_cuda
        value = orig(triples, negatives, slot, offset, batch_size, loss, temperature, dropout=dropout,
                     implementation=implementation)
        if len(checked) < 4:
            e, r = job.model._b200_weights()
            z = nso.block("complex", e.detach().double().cpu(), r.detach().double().cpu(), triples.cpu(), slot,
                          negatives.cpu(), dropout, implementation)
            checked.append((float(value), float(nlo.ns_loss(z, "kl", batch_size=batch_size))))
        return value

    job.model.loss_negatives = spy
    job.epoch += 1
    job._prepare()
    assert math.isfinite(job.run_epoch()["avg_loss"])
    assert len(checked) == 4
    for got, want in checked:
        assert got == pytest.approx(want, rel=TOL)


@needs_ref
@pytest.mark.parametrize("mode", ["dropout0", "eval"])
def test_eval_mode_and_dropout_zero_take_the_existing_kernels(mode, splits):
    import jobs_util as ju
    from kge_b200.plugin.jobs import _fused_model

    p = 0.0 if mode == "dropout0" else 0.3
    cfg = {"b200_complex.entity_embedder.dropout": p, "negative_sampling.num_samples.s": 3,
           "negative_sampling.num_samples.o": 3, "user.b200_ns_dropout": True}
    job = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", train_type="negative_sampling", loss="kl",
                      batch_size=32, forward_only=(mode == "eval"), extra=cfg,
                      job_class="B200TrainingJobNegativeSampling")
    keys = []

    def spy(name):
        orig = getattr(job.model, name)

        def f(*a, **kw):
            keys.append(kw.get("dropout"))
            return orig(*a, **kw)
        return f

    job.model.loss_negatives, job.model.score_negatives = spy("loss_negatives"), spy("score_negatives")
    job.epoch += 1
    job._prepare()
    batch = next(iter(job.loader))
    if mode == "eval":
        job.model.eval()
    assert job.model.b200_dropout_rates() is None and _fused_model(job.model) is job.model
    job._process_batch(0, batch)
    assert keys and all(k is None for k in keys)
