"""The negative-sampling P slot without a GPU: the C ABI of b200kge_ns_p_backward (symbols, argument refusals before any
launch, workspace sizes), the routing of `user.b200_ns_p_slot` in B200TrainingJobNegativeSampling with oracle-backed
engine stand-ins, and two epochs of the option-on job against the reference job.  tests/test_gpu_ns_p_slot.py runs the
kernels."""
import ctypes as C
import os
import re

import pytest
import torch

import ns_loss_oracle as nlo
from kge_b200 import hostenv

S, P, O = 0, 1, 2
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "b200kge.h")


# ---- C ABI
@pytest.fixture(scope="module")
def lib():
    from kge_b200 import _lib

    try:
        return _lib.load()
    except OSError as e:
        pytest.skip(f"libb200kge.so not loadable here: {e}")


def test_header_and_signatures_declare_the_entry():
    from kge_b200 import _lib

    text = open(HEADER).read()
    for name in ("b200kge_ns_p_backward", "b200kge_ns_p_backward_workspace_bytes"):
        assert re.search(rf"\b{name}\(", text), name
        assert name in _lib.SIGNATURES, name
    m = re.search(r"#define B200KGE_NS_P_MAX_RELATIONS (\d+)", text)
    assert m and int(m.group(1)) == _lib.NS_P_MAX_RELATIONS


def _call(lib, **over):
    from kge_b200._lib import Rows

    E, R, D, n, K = 50, 6, 16, 3, 4
    buf = (C.c_float * 16)()
    ids = (C.c_int64 * 64)()
    ent, rel = Rows(), Rows()
    for r, rows, dim in ((ent, E, D), (rel, over.pop("R", R), over.pop("Dr", D))):
        r.base, r.idx, r.rows, r.ld, r.dim = C.addressof(buf), None, rows, D, dim
    a = dict(model=0, l_norm=1.0, ent=ent, rel=rel, triples=C.addressof(ids), neg=C.addressof(ids), n=n, K=K,
             g=C.addressof(buf), ldg=K + 1, es=1, er=C.addressof(ids), ec=C.addressof(ids), de=C.addressof(buf), lde=D,
             rs=1, rr=C.addressof(ids), rcnt=C.addressof(ids), dr=C.addressof(buf), ldr=D, ws=C.addressof(buf), wsb=0)
    a.update(over)
    return lib.b200kge_ns_p_backward(a["model"], a["l_norm"], C.byref(a["ent"]), C.byref(a["rel"]), a["triples"],
                                     a["neg"], a["n"], a["K"], a["g"], a["ldg"], a["es"], a["er"], a["ec"], a["de"],
                                     a["lde"], a["rs"], a["rr"], a["rcnt"], a["dr"], a["ldr"], a["ws"], a["wsb"], None)


def test_entry_refuses_bad_arguments(lib):
    from kge_b200._lib import ERR_INVALID as INVALID, ERR_UNSUPPORTED as UNSUPPORTED, ERR_WORKSPACE as WORKSPACE

    assert _call(lib, g=None) == INVALID                        # grad_scores is required, for BCE too
    assert _call(lib, triples=None) == INVALID
    assert _call(lib, neg=None) == INVALID
    assert _call(lib, er=None) == INVALID                       # sparse entity table without rows
    assert _call(lib, rcnt=None) == INVALID                     # sparse relation table without a count
    assert _call(lib, de=None) == INVALID
    assert _call(lib, ldg=4) == INVALID                         # narrower than the 1 + K columns
    assert _call(lib, lde=8) == INVALID
    assert _call(lib, n=-1) == INVALID
    assert _call(lib, model=9) == INVALID
    assert _call(lib, model=5, l_norm=3.0) == UNSUPPORTED       # TransE L3
    assert _call(lib, model=6, l_norm=2.0, Dr=8) == UNSUPPORTED  # RotatE L2
    assert _call(lib, R=4097) == UNSUPPORTED                    # above B200KGE_NS_P_MAX_RELATIONS
    assert _call(lib, wsb=0) == WORKSPACE
    assert _call(lib, ws=None, wsb=1 << 20) == WORKSPACE
    # dense tables: the row outputs may be null
    assert _call(lib, es=0, er=None, ec=None, rs=0, rr=None, rcnt=None, wsb=0) == WORKSPACE


@pytest.mark.parametrize("model", [0, 4, 5, 6])
def test_workspace_bytes_grow_with_the_problem(lib, model):
    from kge_b200._lib import NS_P_MAX_RELATIONS

    D = 16 if model == 4 else 128

    def ws(n=512, K=100, E=40943, R=237):
        return lib.b200kge_ns_p_backward_workspace_bytes(model, n, K, D, E, R)

    base = ws()
    assert base > 0
    assert ws(n=1024) > base and ws(E=4_800_000) > base and ws(R=1000) > base
    assert ws(n=0) <= base and ws(R=11) <= base
    assert ws(K=1000) >= base                                  # C [n, R] does not depend on K
    assert ws(R=NS_P_MAX_RELATIONS) > 0 and ws(R=NS_P_MAX_RELATIONS + 1) == 0
    assert lib.b200kge_ns_p_backward_workspace_bytes(model, -1, 4, D, 50, 6) == 0


# ---- the job on the CPU (engine stand-ins)
E, R, D = 30, 4, 8


@pytest.fixture()
def splits():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 120, 20, 20)


def _dense_grads(model, ent, rel, triples, slot, neg, grad_scores, l_norm):
    """The oracle's gradient of sum(G * block) for one slot's [n, 1+K] block."""
    from oracle import kge_fold as kf

    d_ent, d_rel = torch.zeros_like(ent), torch.zeros_like(rel)
    n, k = neg.shape
    t = triples.long().repeat_interleave(1 + k, 0).view(n, 1 + k, 3).clone()
    t[:, 1:, slot] = neg.long()
    t = t.view(-1, 3)
    kf.spo_backward(model, ent.detach(), rel.detach(), t[:, 0], t[:, 1], t[:, 2], grad_scores.reshape(-1), d_ent, d_rel,
                    l_norm)
    return d_ent, d_rel


def _as_sparse(x, rows):
    rows = torch.as_tensor(rows, dtype=torch.int64)
    return torch.sparse_coo_tensor(rows[None, :], x[rows], x.shape, is_coalesced=True)


@pytest.fixture()
def stub():
    """tests/engine_stub.py plus oracle-backed ns_loss, ns_backward (grad_scores form), ns_backward_sparse and
    ns_p_backward; counts the calls."""
    import engine_stub
    import ns_sparse_oracle as nsp
    from kge_b200 import engine

    calls = {"ns_loss": 0, "ns_backward": 0, "ns_backward_sparse": 0, "ns_p_backward": 0, "p_sparse": []}
    plain = engine_stub.ns_backward

    def ns_loss(scores, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None, want_grad=False,
                return_rows=False):
        calls["ns_loss"] += 1
        z = scores.detach()
        return (nlo.ns_loss(z, loss, arg, temperature, label_idx, batch_size),
                nlo.ns_loss_grad(z, loss, arg, temperature, label_idx, batch_size) if want_grad else None)

    def ns_backward(model, ent, rel, triples, negatives, offset=0.0, l_norm=1.0, batch_size=None, grad_scores=None):
        calls["ns_backward"] += 1
        if grad_scores is None:
            return plain(model, ent, rel, triples, negatives, offset, l_norm, batch_size)
        d_ent, d_rel = torch.zeros_like(ent), torch.zeros_like(rel)
        for slot, neg in negatives.items():
            de, dr = _dense_grads(model, ent, rel, triples, slot, neg, grad_scores[slot], l_norm)
            d_ent += de
            d_rel += dr
        return d_ent, d_rel

    def ns_backward_sparse(model, ent, rel, triples, slot, negatives, offset=0.0, l_norm=1.0, batch_size=None,
                           grad_scores=None, dropout=None, implementation="batch", sparse=(True, True)):
        calls["ns_backward_sparse"] += 1
        d = _dense_grads(model, ent, rel, triples, slot, negatives, grad_scores, l_norm)
        rows = nsp.row_sets(triples.numpy(), negatives.numpy(), implementation, ent.shape[0])
        return tuple(_as_sparse(x, r) if sp else x for x, r, sp in zip(d, rows, sparse))

    def ns_p_backward(model, ent, rel, triples, negatives, grad_scores, l_norm=1.0, implementation="batch",
                      sparse=(False, False)):
        calls["ns_p_backward"] += 1
        calls["p_sparse"].append(tuple(sparse))
        d_ent, d_rel = _dense_grads(model, ent, rel, triples, P, negatives, grad_scores, l_norm)
        tri = triples.long()
        rows_e = torch.unique(torch.cat((tri[:, 0], tri[:, 2])))
        rows_r = (torch.arange(rel.shape[0]) if implementation == "all"
                  else torch.unique(torch.cat((tri[:, 1], negatives.long().reshape(-1)))))
        return (_as_sparse(d_ent, rows_e) if sparse[0] else d_ent, _as_sparse(d_rel, rows_r) if sparse[1] else d_rel)

    names = ("ns_loss", "ns_backward", "ns_backward_sparse", "ns_p_backward")
    with engine_stub.installed():
        saved = {k: getattr(engine, k) for k in names}
        for k, f in zip(names, (ns_loss, ns_backward, ns_backward_sparse, ns_p_backward)):
            setattr(engine, k, f)
        try:
            yield calls
        finally:
            for k, v in saved.items():
                setattr(engine, k, v)


def _extra(option, loss="kl", impl="triple", **more):
    extra = {"negative_sampling.num_samples.s": 3, "negative_sampling.num_samples.p": 6,
             "negative_sampling.num_samples.o": 4, "negative_sampling.implementation": impl,
             "train.loss_arg": 1.0 if loss.startswith("bce") else 0.5}
    if option:
        extra["user.b200_ns_p_slot"] = True
    extra.update(more)
    return extra


def _train_pair(splits, extra, model="complex", loss="kl", mutate=None):
    """Two epochs of the plugin job (`extra` as given) and of the reference job (without the user.* options) from the
    same tables; keys starting with "M." are the model's options."""
    import jobs_util as ju

    def cfg(tag):
        name = model if tag == "ref" else "b200_" + model
        return {k.replace("M.", name + ".", 1): v for k, v in extra.items()
                if not (tag == "ref" and k.startswith("user."))}

    torch.manual_seed(0)
    init = ju.make_job(model, E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=16,
                       extra=cfg("ref"))
    out = {}
    for tag in ("ref", "plugin"):
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "plugin" else {}
        job = ju.make_job(model if tag == "ref" else "b200_" + model, E, R, D, splits, train_type="negative_sampling",
                          loss=loss, batch_size=16, forward_only=False, extra=cfg(tag), **kw)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a)
        if tag == "plugin" and mutate is not None:
            mutate(job)
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        out[tag] = losses
    return out


@pytest.mark.parametrize("loss", ["kl", "bce", "margin_ranking", "bce_self_adversarial"])
@pytest.mark.parametrize("model", ["complex", "rotate"])
def test_option_on_trains_every_slot_natively(splits, stub, model, loss):
    out = _train_pair(splits, _extra(True, loss), model=model, loss=loss)
    assert stub["ns_p_backward"] > 0 and stub["ns_backward"] > 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
@pytest.mark.parametrize("sparse_ent,sparse_rel", [(True, True), (True, False), (False, True)])
def test_sparse_tables_take_the_row_sparse_p_output(splits, stub, impl, sparse_ent, sparse_rel):
    more = {"M.entity_embedder.sparse": sparse_ent, "M.relation_embedder.sparse": sparse_rel,
            "train.optimizer.default.type": "Adagrad"}
    out = _train_pair(splits, _extra(True, impl=impl, **more))
    assert stub["ns_p_backward"] > 0 and stub["ns_backward_sparse"] > 0, stub
    assert set(stub["p_sparse"]) == {(sparse_ent, sparse_rel)}
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_option_off_changes_nothing(splits, stub):
    out = _train_pair(splits, _extra(False))
    assert stub["ns_p_backward"] == 0 and stub["ns_loss"] == 0 and stub["ns_backward"] == 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def _no_native_route(stub):
    assert stub["ns_p_backward"] == 0 and stub["ns_backward"] == 0 and stub["ns_backward_sparse"] == 0, stub


def test_dropout_keeps_the_reference_step(splits, stub):
    more = {"M.entity_embedder.dropout": 0.2, "M.relation_embedder.dropout": 0.1}
    out = _train_pair(splits, _extra(True, **more))
    _no_native_route(stub)
    assert len(out["plugin"]) == 2


def test_reciprocal_wrapper_keeps_the_reference_step(splits, stub):
    import jobs_util as ju

    extra = _extra(True)
    extra["reciprocal_relations_model.base_model.type"] = "b200_complex"
    job = ju.make_job("reciprocal_relations_model", E, R, D, splits, train_type="negative_sampling", loss="kl",
                      batch_size=16, forward_only=False, extra=extra, imports=("b200_complex",),
                      job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    job._prepare()
    with pytest.raises(Exception):               # the reference's score_so raises for the wrapper
        job.run_epoch()
    _no_native_route(stub)


def test_unserved_norm_keeps_the_reference_step(splits, stub):
    out = _train_pair(splits, _extra(True, **{"M.l_norm": 3.0}), model="transe")
    _no_native_route(stub)
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_reference_backward_keeps_the_reference_step(splits, stub):
    def mutate(job):
        job.model.b200_backward = "reference"
    out = _train_pair(splits, _extra(True), mutate=mutate)
    _no_native_route(stub)
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_too_many_relations_keep_the_reference_step(splits, stub, monkeypatch):
    import kge_b200.plugin as plugin

    monkeypatch.setattr(plugin, "NS_P_MAX_RELATIONS", R - 1)
    out = _train_pair(splits, _extra(True))
    _no_native_route(stub)
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_device_sampling_with_an_unserved_p_slot_still_raises(splits, stub):
    import jobs_util as ju

    extra = _extra(True, **{"user.b200_device_sampling": True, "b200_transe.l_norm": 3.0})
    job = ju.make_job("b200_transe", E, R, D, splits, train_type="negative_sampling", loss="kl", batch_size=16,
                      forward_only=False, extra=extra, job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    job._prepare()
    with pytest.raises(NotImplementedError, match="b200_device_sampling"):
        job.run_epoch()
