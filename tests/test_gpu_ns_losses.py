"""The negative-sampling losses on the H100: the row-loss kernel (b200kge_ns_loss) against the reference's recorded
values and gradients (tests/golden/ns_losses.npz), the G-driven NS backward (b200kge_ns_backward with grad_scores) against the CPU
algebra in fp64, and B200TrainingJobNegativeSampling training with every loss against the reference job."""
import os

import numpy as np
import pytest
import torch

import ns_loss_oracle as nlo
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ns_losses.npz")
S, P, O = 0, 1, 2
TOL = 1e-4
NEW_LOSSES = ["kl", "bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se"]


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    return engine


def _assert_close(got, ref, what, tol=TOL):
    got = got.detach().cpu().double()
    ref = ref.double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    err = float((got - ref).abs().max()) if ref.numel() else 0.0
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


def _golden_cases():
    z = np.load(GOLDEN)
    for j, name in enumerate(z["loss_name"]):
        yield (str(name), float(z["arg"][j]), float(z["temperature"][j]), torch.from_numpy(z[f"z_{j}"]),
               torch.from_numpy(z[f"lab_{j}"]), float(z[f"loss_{j}"]), torch.from_numpy(z[f"grad_{j}"]))


def test_ns_loss_golden(eng):
    """Every loss, offsets / temperatures / margins, K in {1, 7, 1000}, rows with |z| >= 100, positives in column 0
    and elsewhere: loss within 1e-5 relative, G within 1e-4 of rms of the reference's autograd dL/dZ."""
    for name, arg, temp, z, lab, loss, grad in _golden_cases():
        what = f"{name} arg={arg} T={temp} shape={tuple(z.shape)}"
        li = None if bool((lab == 0).all()) else lab.cuda()
        val, G = eng.ns_loss(z.cuda(), name, arg, temp, label_idx=li, want_grad=True)
        assert float(val) == pytest.approx(loss, rel=1e-5, abs=1e-6), what
        _assert_close(G, grad, what)
        # batch_size scales both outputs
        val4, G4 = eng.ns_loss(z.cuda(), name, arg, temp, label_idx=li, batch_size=4, want_grad=True)
        assert float(val4) == pytest.approx(loss / 4, rel=1e-5, abs=1e-6), what
        _assert_close(G4, grad / 4, what)


@pytest.mark.parametrize("loss", nlo.LOSSES)
@pytest.mark.parametrize("n,K", [(1, 1), (37, 30), (64, 1000), (3, 9000)])
def test_ns_loss_deterministic_and_vs_oracle(eng, loss, n, K):
    """Two identical calls give bit-identical loss, row losses and G; rows wider than a block (K = 9000) and the fp64
    restatement agree."""
    if K == 1 and loss in ("bce_mean", "bce_self_adversarial", "margin_ranking"):
        K = 2
    z = torch.randn((n, 1 + K), generator=torch.Generator().manual_seed(n + K)) * 5
    zc = z.cuda()
    a = eng.ns_loss(zc, loss, 0.75, 0.5, batch_size=7, want_grad=True, return_rows=True)
    b = eng.ns_loss(zc, loss, 0.75, 0.5, batch_size=7, want_grad=True, return_rows=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    ref = nlo.ns_loss(z.double(), loss, 0.75, 0.5, batch_size=7)
    assert float(a[0]) == pytest.approx(float(ref), rel=1e-5)
    _assert_close(a[1], nlo.ns_loss_grad(z.double(), loss, 0.75, 0.5, batch_size=7), loss)
    _assert_close(a[2], nlo.ns_loss_rows(z.double(), loss, 0.75, 0.5), loss + " rows")


def test_margin_tie_on_scored_block(eng):
    """A negative id equal to the positive's entity scores like column 0 — to the last bits only: column 0 comes from the
    row-wise triple kernel, the negatives from the folded form — and with margin 0 an exact tie takes the gradient, as
    torch's MarginRankingLoss does (clamp_min passes it at 0)."""
    model, E, R, D, n, K = "complex", 97, 5, 32, 11, 6
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    negs = torch.randint(0, E, (n, K), generator=torch.Generator().manual_seed(5))
    negs[:, 2] = tri[:, O]
    z = eng.ns_score(model, ent.cuda(), rel.cuda(), tri.cuda(), negs.cuda(), O, True)
    assert torch.allclose(z[:, 0], z[:, 3], rtol=1e-6, atol=1e-6)
    z[:, 3] = z[:, 0]                                    # the exact tie
    _, G = eng.ns_loss(z, "margin_ranking", 0.0, want_grad=True)
    G, zz = G.cpu(), z.cpu()
    assert (G[:, 3] == 1.0).all()
    active = ((-(zz[:, :1] - zz[:, 1:])) >= 0).sum(1).float()
    assert torch.equal(G[:, 0], -active)


def test_loss_dense_refuses_row_wise_kinds(eng):
    z = torch.randn(4, 9).cuda()
    lab = torch.zeros(4, dtype=torch.int64).cuda()
    for loss in ("bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se"):
        with pytest.raises(NotImplementedError):
            eng.loss_dense(z, lab, loss)


def test_mirror_kgeloss(eng):
    """kge_b200.model.KgeLoss: create_negative_sampling() resolves the reference's loss_arg defaults; index labels and
    the 0/1 matrix give the same value."""
    from kge_b200.model import KgeLoss

    z = torch.randn((6, 9), generator=torch.Generator().manual_seed(1)) * 3
    lab = torch.tensor([0, 3, 8, 1, 1, 5])
    y = torch.zeros(6, 9)
    y[torch.arange(6), lab] = 1
    for name, arg in (("bce_mean", 0.0), ("bce_self_adversarial", 0.0), ("margin_ranking", 1.0), ("soft_margin", 0.0),
                      ("se", 0.0)):
        loss = KgeLoss.create_negative_sampling(name)
        assert loss._offset == arg
        ref = float(nlo.ns_loss(z.double(), name, arg, 1.0, lab))
        assert float(loss(z.cuda(), lab.cuda())) == pytest.approx(ref, rel=1e-5)
        assert float(loss(z.cuda(), y.cuda())) == pytest.approx(ref, rel=1e-5)
    with pytest.raises(ValueError):
        KgeLoss.create_negative_sampling("se")(z.cuda(), torch.ones(6, 9).cuda())


@pytest.mark.parametrize("loss", nlo.LOSSES)
@pytest.mark.parametrize("model,D,ln", [("complex", 64, 1.0), ("distmult", 32, 1.0), ("simple", 64, 1.0), ("cp", 64, 1.0),
                                        ("rescal", 16, 1.0), ("transe", 64, 1.0), ("transe", 64, 2.0), ("rotate", 64, 1.0)])
def test_ns_backward_grad(eng, loss, model, D, ln):
    """The G-driven NS backward (S and O slots, different K) against the generalised CPU algebra in fp64."""
    E, R, n, K = 501, 5, 37, 150
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    g = torch.Generator().manual_seed(3)
    negs = {S: torch.randint(0, E, (n, K), generator=g), O: torch.randint(0, E, (n, K + 7), generator=g)}
    arg = {"margin_ranking": 1.0, "bce": 0.25, "bce_mean": 0.25, "bce_self_adversarial": 0.25}.get(loss, 0.0)
    bs = 50
    ref_e, ref_r = nlo.ns_backward(model, ent.double(), rel.double(), tri, negs, loss, arg, 0.5, ln, bs)
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    grads = {}
    for slot, neg in negs.items():
        z = eng.ns_score(model, ec, rc, tc, neg.cuda(), slot, True, ln)
        grads[slot] = eng.ns_loss(z, loss, arg, 0.5, batch_size=bs, want_grad=True)[1]
    d_ent, d_rel = eng.ns_backward(model, ec, rc, tc, {k: v.cuda() for k, v in negs.items()}, l_norm=ln,
                                   grad_scores=grads)
    _assert_close(d_ent, ref_e, f"{model} {loss} d_ent")
    _assert_close(d_rel, ref_r, f"{model} {loss} d_rel")


def test_ns_backward_grad_reproduces_bce(eng):
    """G from the row-loss kernel with bce reproduces the kernel's own BCE gradient."""
    model, E, R, D, n, K = "rotate", 301, 5, 64, 29, 40
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n).cuda()
    neg = torch.randint(0, E, (n, K), generator=torch.Generator().manual_seed(8)).cuda()
    ec, rc = ent.cuda(), rel.cuda()
    z = eng.ns_score(model, ec, rc, tri, neg, S, True)
    G = eng.ns_loss(z, "bce", 0.5, batch_size=64, want_grad=True)[1]
    a = eng.ns_backward(model, ec, rc, tri, {S: neg}, 0.5, 1.0, 64)
    b = eng.ns_backward(model, ec, rc, tri, {S: neg}, grad_scores={S: G})
    _assert_close(b[0], a[0].cpu(), "d_ent")
    _assert_close(b[1], a[1].cpu(), "d_rel")


# ------------------------------------------------------------------------------------------------------------ job level
JE, JR, JD = 211, 5, 32


@pytest.fixture(scope="module")
def splits():
    from kge_b200 import hostenv

    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _extra(loss):
    extra = {"negative_sampling.num_samples.s": 11, "negative_sampling.num_samples.o": 13,
             "negative_sampling.implementation": "triple"}
    if loss.startswith("bce"):
        extra["train.loss_arg"] = 1.0
    if loss == "bce_self_adversarial":
        extra["user.bce_self_adversarial_temperature"] = 0.5
    return extra


@pytest.mark.parametrize("loss", NEW_LOSSES)
@pytest.mark.parametrize("model", ["complex", "transe", "rotate"])
def test_ns_job_training_native(model, loss, splits, monkeypatch):
    """Two training epochs (forward, the G-driven backward, Adagrad) track the reference job on the CPU, which draws the
    same negatives; the reference's recompute route is disabled so the native route must have run."""
    import jobs_util as ju
    from kge_b200 import engine, hostenv

    hostenv.import_kge()                                 # the plugin imports the reference's model classes
    from kge_b200.plugin import _B200ModelMixin

    def no_recompute(*a, **kw):
        raise AssertionError("the recompute backward ran")

    monkeypatch.setattr(_B200ModelMixin, "_b200_ref_scores", no_recompute)
    extra = _extra(loss)
    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, device="cpu", train_type="negative_sampling", loss=loss,
                       batch_size=64, extra=extra)
    losses = {}
    for tag, dev in (("ref", "cpu"), ("native", "cuda")):
        name = model if tag == "ref" else "b200_" + model
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "native" else {}
        job = ju.make_job(name, JE, JR, JD, splits, device=dev, train_type="negative_sampling", loss=loss,
                          batch_size=64, forward_only=False, extra=extra, **kw)
        ju.copy_tables(init, job)
        engine.launch_count(reset=True)
        out = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            out.append(job.run_epoch()["avg_loss"])
        if tag == "native":
            assert engine.launch_count() > 0
        losses[tag] = out
    assert losses["native"][0] == pytest.approx(losses["ref"][0], rel=1e-4)
    assert losses["native"][1] == pytest.approx(losses["ref"][1], rel=1e-3)


@pytest.mark.parametrize("loss", NEW_LOSSES)
def test_ns_job_forward_only(loss, splits):
    import jobs_util as ju

    extra = _extra(loss)
    torch.manual_seed(0)
    ref = ju.make_job("complex", JE, JR, JD, splits, device="cpu", train_type="negative_sampling", loss=loss,
                      batch_size=64, extra=extra)
    dev = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", train_type="negative_sampling", loss=loss,
                      batch_size=64, extra=extra, job_class="B200TrainingJobNegativeSampling")
    ju.copy_tables(ref, dev)
    a = ju.run_forward_epoch(ref)["avg_loss"]
    assert ju.run_forward_epoch(dev)["avg_loss"] == pytest.approx(a, rel=1e-4)
    dev._max_subbatch_size = 10
    assert ju.run_forward_epoch(dev)["avg_loss"] == pytest.approx(a, rel=1e-4)


def test_ns_job_device_sampling_with_kl(splits):
    """user.b200_device_sampling with kl: negatives drawn on the device, training runs natively."""
    import jobs_util as ju

    extra = dict(_extra("kl"), **{"user.b200_device_sampling": True})
    torch.manual_seed(0)
    job = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", train_type="negative_sampling", loss="kl",
                      batch_size=64, forward_only=False, extra=extra, job_class="B200TrainingJobNegativeSampling")
    assert job._device_sampling
    job.epoch += 1
    job._prepare()
    ju.seed_all(3)
    a = job.run_epoch()["avg_loss"]
    job.epoch += 1
    b = job.run_epoch()["avg_loss"]
    assert job._sample_calls > 0
    assert np.isfinite(a) and np.isfinite(b) and a > 0 and b > 0
