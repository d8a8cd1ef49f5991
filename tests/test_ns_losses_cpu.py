"""The negative-sampling losses on the CPU: the restatement (tests/ns_loss_oracle.py) against the reference's KgeLoss
classes — recorded (tests/golden/ns_losses.npz) and, where the reference is installed, live on fresh seeds — and the
routing of the job plugin: B200TrainingJobNegativeSampling trains every loss through the native slot node, while the P
slot and the 1vsAll / KvsAll jobs fall through to the reference for these losses.  kge_b200.engine is replaced by
oracle-backed stand-ins here; tests/test_gpu_ns_losses.py runs the kernels."""
import os

import numpy as np
import pytest
import torch

import ns_loss_oracle as nlo
from oracle import ref_shim

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ns_losses.npz")
REL = 2e-6


def _golden_cases():
    z = np.load(GOLDEN)
    for j, name in enumerate(z["loss_name"]):
        yield (str(name), float(z["arg"][j]), float(z["temperature"][j]), torch.from_numpy(z[f"z_{j}"]),
               torch.from_numpy(z[f"lab_{j}"]), float(z[f"loss_{j}"]), torch.from_numpy(z[f"grad_{j}"]))


def test_golden_covers_the_issue_grid():
    cases = list(_golden_cases())
    assert {c[0] for c in cases} == set(nlo.LOSSES)
    assert {c[3].shape[1] - 1 for c in cases} == {1, 7, 1000}
    assert any(c[3].abs().min() >= 100 for c in cases)
    assert {c[1] for c in cases if c[0] == "margin_ranking"} == {0.0, 1.0}
    assert {c[2] for c in cases if c[0] == "bce_self_adversarial"} == {0.5, 1.0}
    assert {c[1] for c in cases if c[0] == "bce_mean"} == {0.0, 2.0}


def test_oracle_matches_golden():
    for name, arg, temp, z, lab, loss, grad in _golden_cases():
        what = f"{name} arg={arg} T={temp} shape={tuple(z.shape)}"
        got = float(nlo.ns_loss(z.double(), name, arg, temp, lab))
        assert got == pytest.approx(loss, rel=REL, abs=1e-12), what
        g = nlo.ns_loss_grad(z.double(), name, arg, temp, lab)
        scale = max(float(grad.double().abs().max()), 1e-12)
        assert float((g - grad.double()).abs().max()) <= REL * scale, what
        # fp32 restatement: the stable forms keep |z| >= 100 finite
        g32 = nlo.ns_loss_grad(z, name, arg, temp, lab)
        assert torch.isfinite(nlo.ns_loss(z, name, arg, temp, lab)) and torch.isfinite(g32).all(), what


def test_margin_tie_takes_the_gradient():
    """torch's clamp_min passes the gradient at exactly 0: margin 0 and a negative equal to the positive."""
    z = torch.tensor([[1.0, 1.0, 0.5, 3.0]])
    g = nlo.ns_loss_grad(z, "margin_ranking", 0.0)
    assert g.tolist() == [[-2.0, 1.0, 0.0, 1.0]]
    x = torch.tensor([1.0], requires_grad=True)
    y = torch.tensor([1.0], requires_grad=True)
    torch.nn.MarginRankingLoss(margin=0.0)(x, y, torch.ones(1)).backward()
    assert (float(x.grad), float(y.grad)) == (-1.0, 1.0)


@pytest.mark.skipif(not ref_shim.available(), reason="reference not installed (oracle/install_ref.sh)")
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_live_reference(dtype):
    ref_shim.import_reference()
    from kge import Config
    from kge.util.loss import KgeLoss

    g = torch.Generator().manual_seed(99)
    for name in nlo.LOSSES:
        for K, arg, temp in ((3, 0.0, 1.0), (40, 1.5, 0.25), (257, 0.0, 2.0)):
            c = Config()
            c.folder = None
            c.set("console.quiet", True)
            c.set("job.device", "cpu")
            c.set("train.type", "negative_sampling")
            c.set("train.loss", name)
            c.set("train.loss_arg", arg)
            c.set("user.bce_self_adversarial_temperature", temp, create=True)
            n = 5
            z = (torch.randn((n, 1 + K), generator=g) * 4).to(dtype).requires_grad_(True)
            y = torch.zeros((n, 1 + K), dtype=dtype)
            y[:, 0] = 1
            value = KgeLoss.create(c)(z, y, num_negatives=K)
            (grad,) = torch.autograd.grad(value, z)
            a = arg if name != "kl" and name != "soft_margin" and name != "se" else 0.0
            t = temp if name == "bce_self_adversarial" else 1.0
            tol = 2e-6 if dtype == torch.float64 else 2e-5
            assert float(nlo.ns_loss(z.detach(), name, a, t)) == pytest.approx(float(value.detach()), rel=tol), (name, K)
            mine = nlo.ns_loss_grad(z.detach(), name, a, t)
            assert float((mine - grad).abs().max()) <= tol * max(float(grad.abs().max()), 1e-12), (name, K)


# ------------------------------------------------------------------------------------------------ job plugin routing
E, R, D = 53, 4, 16


@pytest.fixture(scope="module")
def splits():
    from kge_b200 import hostenv

    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 150, 20, 20)


@pytest.fixture()
def stub():
    """tests/engine_stub.py plus oracle-backed ns_loss and the grad_scores form of ns_backward; counts their calls."""
    import engine_stub
    from kge_b200 import engine

    calls = {"ns_loss": 0, "ns_backward_grad": 0}
    plain_backward = engine_stub.ns_backward

    def ns_loss(scores, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None, want_grad=False,
                return_rows=False):
        calls["ns_loss"] += 1
        z = scores.detach()
        value = nlo.ns_loss(z, loss, arg, temperature, label_idx, batch_size)
        return value, (nlo.ns_loss_grad(z, loss, arg, temperature, label_idx, batch_size) if want_grad else None)

    def ns_backward(model, ent, rel, triples, negatives, offset=0.0, l_norm=1.0, batch_size=None, grad_scores=None):
        if grad_scores is None:
            return plain_backward(model, ent, rel, triples, negatives, offset, l_norm, batch_size)
        calls["ns_backward_grad"] += 1
        from oracle import kge_fold as kf

        d_ent, d_rel = torch.zeros_like(ent), torch.zeros_like(rel)
        n = triples.shape[0]
        for slot, neg in negatives.items():      # G is given: scatter it through the row-wise backward
            k = neg.shape[1]
            t = triples.long().repeat_interleave(1 + k, 0).view(n, 1 + k, 3).clone()
            t[:, 1:, slot] = neg.long()
            t = t.view(-1, 3)
            kf.spo_backward(model, ent.detach(), rel.detach(), t[:, 0], t[:, 1], t[:, 2],
                            grad_scores[slot].reshape(-1), d_ent, d_rel, l_norm)
        return d_ent, d_rel

    with engine_stub.installed():
        saved = engine.ns_loss, engine.ns_backward
        engine.ns_loss, engine.ns_backward = ns_loss, ns_backward
        try:
            yield calls
        finally:
            engine.ns_loss, engine.ns_backward = saved


def _extra(loss, p_samples=0):
    extra = {"negative_sampling.num_samples.s": 5, "negative_sampling.num_samples.o": 6,
             "negative_sampling.num_samples.p": p_samples, "negative_sampling.implementation": "triple"}
    if loss == "margin_ranking":
        extra["train.loss_arg"] = 0.5
    if loss.startswith("bce"):
        extra["train.loss_arg"] = 1.0
    if loss == "bce_self_adversarial":
        extra["user.bce_self_adversarial_temperature"] = 0.5
    return extra


def _two_epochs(job):
    import jobs_util as ju

    out = []
    for ep in range(2):
        job.epoch += 1
        if job.loader is None:
            job._prepare()
        ju.seed_all(10 + ep)
        out.append(job.run_epoch()["avg_loss"])
    return out


def _train_pair(loss, splits, p_samples=0):
    import jobs_util as ju

    torch.manual_seed(0)
    extra = _extra(loss, p_samples)
    init = ju.make_job("complex", E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=16, extra=extra)
    out = {}
    for tag in ("ref", "plugin"):
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "plugin" else {}
        job = ju.make_job("complex" if tag == "ref" else "b200_complex", E, R, D, splits, train_type="negative_sampling",
                          loss=loss, batch_size=16, forward_only=False, extra=extra, **kw)
        ju.copy_tables(init, job)
        out[tag] = _two_epochs(job)
    return out


@pytest.mark.parametrize("loss", ["kl", "bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se"])
def test_ns_job_trains_natively(loss, splits, stub):
    out = _train_pair(loss, splits)
    assert stub["ns_loss"] > 0 and stub["ns_backward_grad"] > 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_ns_job_p_slot_falls_through(splits, stub):
    out = _train_pair("kl", splits, p_samples=2)
    assert stub["ns_loss"] == 0 and stub["ns_backward_grad"] == 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_loss_classifiers(splits):
    import jobs_util as ju
    from kge_b200.plugin import jobs

    for loss in nlo.LOSSES:
        job = ju.make_job("complex", E, R, D, splits, train_type="negative_sampling", loss=loss, extra=_extra(loss))
        kind = jobs._ns_loss_kind(job.loss)
        assert kind is not None and kind[0] == loss
        if loss == "margin_ranking":
            assert kind[1] == 0.5
        if loss == "bce_self_adversarial":
            assert kind[1:] == (1.0, 0.5)
        # the 1vsAll / KvsAll steps keep their bce / kl scope: every other loss runs the reference's step there
        assert (jobs._fused_loss_kind(job.loss) is None) == (loss not in ("bce", "kl"))


def test_1vsall_job_falls_through_for_soft_margin(splits, stub):
    import jobs_util as ju

    torch.manual_seed(0)
    ref = ju.make_job("complex", E, R, D, splits, loss="soft_margin", batch_size=32)
    fused = ju.make_job("b200_complex", E, R, D, splits, loss="soft_margin", batch_size=32,
                        job_class="B200TrainingJob1vsAll")
    ju.copy_tables(ref, fused)
    a = ju.run_forward_epoch(ref)["avg_loss"]
    assert ju.run_forward_epoch(fused)["avg_loss"] == pytest.approx(a, rel=1e-5)
    assert stub["ns_loss"] == 0
