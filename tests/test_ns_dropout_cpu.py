"""Embedding dropout of the negative-sampling job on CPU: properties of the NS mask layout on the mirror
(tests/ns_dropout_oracle.py) and the job plugin's routing of `user.b200_ns_dropout`.  The kernels are checked against
the same mirror, and the job against the reference job drawing the mirror's masks, in tests/test_gpu_ns_dropout.py."""
import math

import pytest
import torch

import dropout_oracle as dro
import ns_dropout_oracle as nso
from kge_b200 import engine, hostenv

E, R, D = 53, 4, 16
P_ENT, P_REL = 0.3, 0.1
KEY = engine.DropoutKey(0.5, 0.5, 4242, 3, 2)


# ---- the mask layout -------------------------------------------------------------------------------------------------
def test_streams_are_disjoint_from_the_1vsall_draws():
    streams = [nso.stream(slot, j) for slot in (0, 2) for j in range(6)]
    assert len(set(streams)) == 12 and min(streams) == 6
    assert all(not 12 <= s < 18 for s in streams)          # the P slot's streams are reserved


def test_triple_rows_are_distinct_per_negative():
    n, K = 3, 4
    rows = (KEY.row_base + torch.arange(n)).repeat_interleave(K) * K + torch.arange(K).repeat(n)
    assert len(set(rows.tolist())) == n * K
    x = torch.ones(n * K, D)
    m = nso.apply_rows(x, 0.5, KEY, nso.stream(2, 5), rows)
    assert not torch.equal(m[0], m[1])                      # the same entity in two triples gets two masks


def test_batch_shares_one_mask_per_entity_id():
    ent = torch.randn(E, D, dtype=torch.float64)
    rel = torch.randn(R, D, dtype=torch.float64)
    tri = torch.tensor([[1, 0, 2], [3, 1, 4]])
    neg = torch.tensor([[5, 5, 7], [7, 5, 9]])                # repeats within and across rows
    b = nso.block("distmult", ent, rel, tri, 2, neg, KEY, "batch")
    # the O slot of `batch`: the score of (s_i, p_i, id) only depends on the row and the id
    x = nso.apply_rows(ent[tri[:, 0]], KEY.p_ent, KEY, nso.stream(2, 3), torch.arange(2) + KEY.row_base)
    r = nso.apply_rows(rel[tri[:, 1]], KEY.p_rel, KEY, nso.stream(2, 4), torch.arange(2) + KEY.row_base)
    t = nso.apply_rows(ent, KEY.p_ent, KEY, nso.stream(2, 5), torch.arange(E))
    want = ((x * r) @ t.T).gather(1, neg)
    assert torch.allclose(b[:, 1:], want)
    assert b[0, 1] == b[0, 2]
    # `triple` draws a fresh mask per corrupted triple
    bt = nso.block("distmult", ent, rel, tri, 2, neg, KEY, "triple")
    assert bt[0, 1] != bt[0, 2]


def test_masks_follow_the_global_row():
    tri = torch.tensor([[1, 0, 2], [3, 1, 4], [0, 2, 6]])
    neg = torch.tensor([[5, 6], [7, 8], [9, 10]])
    ent = torch.randn(E, D, dtype=torch.float64)
    rel = torch.randn(R, D, dtype=torch.float64)
    for impl in ("triple", "batch"):
        full = nso.block("complex", ent, rel, tri, 0, neg, KEY._replace(row_base=0), impl)
        tail = nso.block("complex", ent, rel, tri[1:], 0, neg[1:], KEY._replace(row_base=1), impl)
        assert torch.allclose(full[1:], tail)                # a sub-batch draws the rows of the whole batch


# ---- job routing ------------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 150, 20, 20)


def _job(model, splits, extra=None, loss="kl"):
    import jobs_util as ju

    cfg = {f"{model}.entity_embedder.dropout": P_ENT, f"{model}.relation_embedder.dropout": P_REL,
           "negative_sampling.num_samples.s": 3, "negative_sampling.num_samples.o": 3}
    cfg.update(extra or {})
    job = ju.make_job(model, E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=32,
                      forward_only=False, extra=cfg, job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    return job


@pytest.fixture()
def stub():
    with nso.installed():
        nso.calls["dropout"] = 0
        yield


def _refuse(*a, **kw):
    raise AssertionError("the native NS step must not run")


@needs_ref
def test_option_off_keeps_the_reference_step(splits, stub):
    job = _job("b200_complex", splits)
    job.model.loss_negatives = job.model.score_negatives = _refuse
    job._prepare()
    assert math.isfinite(job.run_epoch()["avg_loss"])


@needs_ref
def test_p_slot_keeps_the_reference_step(splits, stub):
    job = _job("b200_complex", splits, {"user.b200_ns_dropout": True, "negative_sampling.num_samples.p": 2})
    job.model.loss_negatives = job.model.score_negatives = _refuse
    job._prepare()
    assert math.isfinite(job.run_epoch()["avg_loss"])


@needs_ref
@pytest.mark.parametrize("extra", [{"negative_sampling.num_samples.p": 2}, {"b200_transe.l_norm": 3.0}])
def test_device_sampling_with_an_unserved_configuration_raises(splits, extra, stub):
    model = "b200_transe" if "b200_transe.l_norm" in extra else "b200_complex"
    job = _job(model, splits, {"user.b200_ns_dropout": True, "user.b200_device_sampling": True, **extra})
    job._prepare()
    with pytest.raises(NotImplementedError, match="b200_ns_dropout"):
        job.run_epoch()


@needs_ref
@pytest.mark.parametrize("subbatch", [None, 10])
def test_forward_and_backward_of_a_slot_share_one_key_per_subbatch(splits, subbatch, stub):
    """The route hands every slot of a sub-batch the same key (the slots draw disjoint streams under it), the forward
    and the backward of a slot run under that key, and each sub-batch gets a fresh key."""
    from kge_b200.plugin import _NsSlotLossFn

    job = _job("b200_complex", splits, {"user.b200_ns_dropout": True, "negative_sampling.implementation": "batch"})
    if subbatch:
        job._max_subbatch_size = subbatch
    seen = []

    def fake(ent_w, rel_w, model, triples, negatives, slot, offset, batch_size, loss, temperature, dropout, impl):
        seen.append((slot, dropout, impl, len(triples)))
        return (ent_w.sum() + rel_w.sum()) * 0.0

    orig = _NsSlotLossFn.apply
    _NsSlotLossFn.apply = fake
    try:
        job._prepare()
        job.run_epoch()
    finally:
        _NsSlotLossFn.apply = orig
    assert seen and all(d is not None and impl == "batch" for _, d, impl, _ in seen)
    keys = [d for _, d, _, _ in seen]
    assert all(a == b for a, b in zip(keys[::2], keys[1::2]))       # S and O of one sub-batch
    assert len({k.call for k in keys[::2]}) == len(keys) // 2       # fresh per sub-batch
    assert keys[0].seed == torch.initial_seed() and keys[0][:2] == pytest.approx((P_ENT, P_REL))
    if subbatch:
        assert sorted({k.row_base for k in keys}) == list(range(0, 32, subbatch))


@needs_ref
def test_route_needs_active_dropout_and_a_native_loss(splits, stub):
    from kge_b200.plugin.jobs import _ns_loss_kind

    job = _job("b200_complex", splits, {"user.b200_ns_dropout": True})
    job._prepare()
    slots = [0, 2]
    assert job._b200_ns_dropout_route(_ns_loss_kind(job.loss), slots)[0] is job.model
    assert job._b200_ns_dropout_route(None, slots) == (None, None)
    job.model.eval()
    assert job._b200_ns_dropout_route(_ns_loss_kind(job.loss), slots) == (None, None)
    assert dro.scale(P_ENT) == pytest.approx(1 / (1 - P_ENT))


def _train_pair(model, splits, impl, Kn, loss, subbatch):
    """Two training epochs of the reference job (mirror masks patched in) and of the plugin job with the option, from
    the same tables; the plugin's engine calls are the CPU stand-ins of tests/ns_dropout_oracle.py."""
    import jobs_util as ju

    # plain SGD: Adagrad's first step divides each gradient element by its own magnitude, which turns fp32 rounding
    # differences on near-zero elements (TransE's sign gradient) into full-size steps
    extra = {"negative_sampling.implementation": impl, "negative_sampling.num_samples.s": Kn,
             "negative_sampling.num_samples.o": Kn, "train.optimizer.default.type": "SGD",
             "train.optimizer.default.args.lr": 0.1}
    torch.manual_seed(0)
    init = ju.make_job(model, E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=32, extra=extra)
    out = {}
    for tag in ("ref", "plugin"):
        m = model if tag == "ref" else "b200_" + model
        cfg = {f"{m}.entity_embedder.dropout": P_ENT, f"{m}.relation_embedder.dropout": P_REL, **extra}
        if tag == "plugin":
            cfg["user.b200_ns_dropout"] = True
        job = ju.make_job(m, E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=32,
                          forward_only=False, extra=cfg,
                          job_class="B200TrainingJobNegativeSampling" if tag == "plugin" else None)
        if tag == "ref":
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
        out[tag] = (losses, job.model.get_s_embedder()._embeddings.weight.detach().clone())
    return out


@needs_ref
@pytest.mark.parametrize("subbatch", [None, 10])
@pytest.mark.parametrize("loss", ["kl", "margin_ranking"])
@pytest.mark.parametrize("impl,Kn", [("triple", 3), ("batch", 40)])
@pytest.mark.parametrize("model", ["complex", "transe"])
def test_plugin_job_matches_the_reference_job(model, impl, Kn, loss, subbatch, splits, stub):
    out = _train_pair(model, splits, impl, Kn, loss, subbatch)
    assert nso.calls["dropout"] > 0                        # the dropout route ran
    assert out["plugin"][0] == pytest.approx(out["ref"][0], rel=1e-4)
    err = float((out["plugin"][1] - out["ref"][1]).abs().max())
    assert err <= 1e-4 * float(out["ref"][1].abs().max())
