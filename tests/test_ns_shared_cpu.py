"""Shared negative sampling without a GPU: a numpy mirror of the column map u(i, c) of b200kge_ns_shared_score checked
against the reference's own samples() over many seeded draws, the collapse C = sum of G per shared id checked against
autograd through the reference's score(), the C ABI's refusals, the routing of `user.b200_ns_shared` in
B200TrainingJobNegativeSampling with oracle-backed engine stand-ins, and the naive sub-batch fix.
tests/test_gpu_ns_shared.py runs the kernels."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import ns_loss_oracle as nlo
from kge_b200 import hostenv

S, P, O = 0, 1, 2
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "b200kge.h")
E, R, D = 30, 4, 8


# ---- mirrors of the kernels' index arithmetic
def u_map(n, K, U, repeat, drop):
    """[n, K]: u(i, c) = (j == drop[i]) ? U : j with j = c < U ? c : repeat[c - U] (drop None: u = j)."""
    j = np.concatenate([np.arange(U, dtype=np.int64), np.asarray(repeat, dtype=np.int64).reshape(-1)])
    assert j.size == K
    if drop is None:
        return np.broadcast_to(j, (n, K)).copy()
    drop = np.asarray(drop, dtype=np.int64).reshape(-1, 1)
    return np.where(j[None, :] == drop, U, j[None, :])


def collapse(G, u, nu):
    """C [n, U']: C[i, u] = the sum of G[i, 1 + c] over the columns c with u(i, c) = u, in column order."""
    n, K = u.shape
    C_ = np.zeros((n, nu), dtype=G.dtype)
    for i in range(n):
        for c in range(K):
            C_[i, u[i, c]] += G[i, 1 + c]
    return C_


def used_ids(unique, drop, n):
    """The shared ids some row uses (the `triple` row set): unique[u] is unused exactly when every row drops u."""
    unique = np.asarray(unique)
    if drop is None:
        return unique
    cnt = np.bincount(np.asarray(drop), minlength=unique.size)
    return unique[cnt < n]


def shared_operands(sm):
    """(unique, repeat, drop, U) of a reference shared sample."""
    drop = getattr(sm, "_drop_index", None)
    unique = sm._unique_samples
    U = unique.numel() - (1 if drop is not None else 0)
    return unique, sm._repeat_indexes.long().reshape(-1), drop, U


@pytest.fixture(scope="module")
def kge():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    hostenv.import_kge()
    import kge.util.sampler as sampler

    return sampler


@pytest.fixture()
def splits():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 120, 20, 20)


def _sampler(splits, shared_type, replacement, impl="batch"):
    import jobs_util as ju

    extra = {"negative_sampling.shared": True, "negative_sampling.shared_type": shared_type,
             "negative_sampling.with_replacement": replacement, "negative_sampling.implementation": impl}
    job = ju.make_job("complex", E, R, D, splits, train_type="negative_sampling", loss="kl", batch_size=16, extra=extra)
    return job._sampler


@pytest.mark.parametrize("replacement", [True, False])
@pytest.mark.parametrize("shared_type", ["naive", "default"])
def test_u_map_reproduces_the_reference_samples(splits, kge, shared_type, replacement):
    import jobs_util as ju

    sm = _sampler(splits, shared_type, replacement)
    tri = splits["train"].long()
    seen_no_drop = 0
    for seed in range(40):
        ju.seed_all(seed)
        n = [1, 3, 16, 40][seed % 4]
        K = [1, 7, 12, 29][(seed // 4) % 4]
        if not replacement and K > E - 1:
            continue
        sample = sm._sample_shared(tri[:n], seed % 2 * 2, K)
        unique, repeat, drop, U = shared_operands(sample)
        u = u_map(n, K, U, repeat.numpy(), None if drop is None else drop.numpy())
        ref = sample.samples()
        assert torch.equal(unique[torch.from_numpy(u)], ref), (seed, n, K)
        # a sub-batch: the rows of drop_index sliced, unique and repeat the batch's
        if n >= 3:
            sl = slice(1, n - 1)
            du = u_map(n - 2, K, U, repeat.numpy(), None if drop is None else drop[sl].numpy())
            assert torch.equal(unique[torch.from_numpy(du)], ref[sl])
            if shared_type == "default":
                assert torch.equal(unique[torch.from_numpy(du)], sample.samples(sl))
        if drop is not None:
            seen_no_drop += int((drop == U).sum())
    if shared_type == "default":
        assert seen_no_drop > 0            # rows that keep every shared sample (drop_index == U) were covered


def test_u_map_rows_without_a_drop():
    # drop == U: the row keeps all U samples, the extra id is unused; drop == 1: every column of sample 1 moves to U
    u = u_map(2, 5, 3, [1, 1], [3, 1])
    assert u.tolist() == [[0, 1, 2, 1, 1], [0, 3, 2, 3, 3]]


class _Unique(torch.nn.Module):
    """A model whose score_sp / score_po return a leaf Z [n, U'] (the scores against the shared rows)."""

    def __init__(self, Z):
        super().__init__()
        self.Z = Z

    def score_sp(self, s, p, o=None):
        return self.Z

    def score_po(self, p, o, s=None):
        return self.Z


@pytest.mark.parametrize("shared_type", ["naive", "default"])
def test_collapse_is_the_gradient_through_the_reference_score(splits, kge, shared_type):
    import jobs_util as ju

    sm = _sampler(splits, shared_type, True, impl="batch")
    tri = splits["train"].long()
    for seed in range(12):
        ju.seed_all(100 + seed)
        n, K = [1, 5, 16][seed % 3], [3, 9, 25][(seed // 3) % 3]
        sample = sm._sample_shared(tri[:n], O, K)
        unique, repeat, drop, U = shared_operands(sample)
        nu = unique.numel()
        Z = torch.randn(n, nu, requires_grad=True)          # float32: the reference's block is torch.empty
        G = torch.randn(n, 1 + K)
        scores = sample.score(_Unique(Z))                  # DefaultSharedNegativeSample / NaiveSharedNegativeSample
        (scores * G[:, 1:]).sum().backward()
        u = u_map(n, K, U, repeat.numpy(), None if drop is None else drop.numpy())
        np.testing.assert_allclose(collapse(G.numpy(), u, nu), Z.grad.numpy(), rtol=1e-6, atol=1e-6)
        # the scores themselves are the assembled block
        np.testing.assert_array_equal(np.take_along_axis(Z.detach().numpy(), u, 1), scores.detach().numpy())


def test_used_ids_mirror():
    assert used_ids([5, 6, 7], [0, 0], 2).tolist() == [6, 7]         # sample 0 dropped by every row
    assert used_ids([5, 6, 7], [2, 2], 2).tolist() == [5, 6]         # no row drops: the extra id is unused
    assert used_ids([5, 6, 7], [0, 2], 2).tolist() == [5, 6, 7]
    assert used_ids([5, 6], None, 4).tolist() == [5, 6]


# ---- C ABI
@pytest.fixture(scope="module")
def lib():
    from kge_b200 import _lib

    try:
        return _lib.load()
    except OSError as e:
        pytest.skip(f"libb200kge.so not loadable here: {e}")


def test_header_and_signatures_declare_the_entries():
    from kge_b200 import _lib

    text = open(HEADER).read()
    for name in ("b200kge_ns_shared_score", "b200kge_ns_shared_score_workspace_bytes", "b200kge_ns_shared_backward",
                 "b200kge_ns_shared_backward_workspace_bytes"):
        assert re.search(rf"\b{name}\(", text), name
        assert name in _lib.SIGNATURES, name


def _tables(over):
    from kge_b200._lib import Rows

    buf = (C.c_float * 64)()
    ent, rel = Rows(), Rows()
    for r, rows, dim in ((ent, over.pop("E", 50), over.pop("D", 16)), (rel, 6, over.pop("Dr", 16))):
        r.base, r.idx, r.rows, r.ld, r.dim = C.addressof(buf), None, rows, 16, dim
    return buf, ent, rel


def _score(lib, **over):
    buf, ent, rel = _tables(over)
    ids = (C.c_int64 * 64)()
    a = dict(model=0, l_norm=1.0, prec=0, triples=C.addressof(ids), slot=2, unique=C.addressof(ids), nu=4,
             repeat=C.addressof(ids), drop=C.addressof(ids), n=3, K=5, impl=1, out=C.addressof(buf), ldo=6, z=None,
             ldz=0, ws=C.addressof(buf), wsb=0)
    a.update(over)
    return lib.b200kge_ns_shared_score(a["model"], a["l_norm"], a["prec"], C.byref(ent), C.byref(rel), a["triples"],
                                       a["slot"], a["unique"], a["nu"], a["repeat"], a["drop"], a["n"], a["K"],
                                       a["impl"], a["out"], a["ldo"], a["z"], a["ldz"], a["ws"], a["wsb"], None)


def _backward(lib, **over):
    buf, ent, rel = _tables(over)
    ids = (C.c_int64 * 64)()
    a = dict(model=0, l_norm=1.0, triples=C.addressof(ids), slot=2, unique=C.addressof(ids), nu=4,
             repeat=C.addressof(ids), drop=C.addressof(ids), n=3, K=5, impl=1, z=None, ldz=0, g=C.addressof(buf),
             ldg=6, es=1, er=C.addressof(ids), ec=C.addressof(ids), de=C.addressof(buf), lde=16, rs=0, rr=None,
             rcnt=None, dr=C.addressof(buf), ldr=16, ws=C.addressof(buf), wsb=0)
    a.update(over)
    return lib.b200kge_ns_shared_backward(a["model"], a["l_norm"], C.byref(ent), C.byref(rel), a["triples"], a["slot"],
                                          a["unique"], a["nu"], a["repeat"], a["drop"], a["n"], a["K"], a["impl"],
                                          a["z"], a["ldz"], a["g"], a["ldg"], a["es"], a["er"], a["ec"], a["de"],
                                          a["lde"], a["rs"], a["rr"], a["rcnt"], a["dr"], a["ldr"], a["ws"], a["wsb"],
                                          None)


@pytest.mark.parametrize("call", ["score", "backward"])
def test_entries_refuse_bad_arguments(lib, call):
    from kge_b200._lib import ERR_INVALID as INVALID, ERR_UNSUPPORTED as UNSUPPORTED, ERR_WORKSPACE as WORKSPACE

    f = _score if call == "score" else _backward
    assert f(lib, triples=None) == INVALID
    assert f(lib, unique=None) == INVALID
    assert f(lib, repeat=None) == INVALID                        # K = 5 > U = 3 needs repeats
    assert f(lib, repeat=None, K=3) == WORKSPACE                 # ... and K = U does not
    assert f(lib, nu=7) == INVALID                               # default: U = 6 > K
    assert f(lib, nu=1) == INVALID                               # default: U = 0 < K
    assert f(lib, drop=None, nu=6) == INVALID                    # naive: U = 6 > K
    assert f(lib, n=-1) == INVALID
    assert f(lib, impl=2) == INVALID
    assert f(lib, model=9) == INVALID
    assert f(lib, slot=1) == UNSUPPORTED                          # the P slot
    assert f(lib, model=5, l_norm=3.0) == UNSUPPORTED             # TransE L3
    assert f(lib, model=6, l_norm=2.0, Dr=8) == UNSUPPORTED       # RotatE L2
    assert f(lib, model=1, D=2048, Dr=2048) == UNSUPPORTED        # folded width above 1024
    assert f(lib, wsb=0) == WORKSPACE
    if call == "score":
        assert f(lib, ldo=5) == INVALID                          # narrower than 1 + K
        assert f(lib, out=None) == INVALID
        assert f(lib, z=C.addressof((C.c_float * 64)()), ldz=3) == INVALID   # narrower than U' = 4
        assert f(lib, prec=3) == UNSUPPORTED                     # tf32
        assert f(lib, prec=5, model=5) == UNSUPPORTED            # f16x3 for a distance model
    else:
        assert f(lib, ldg=5) == INVALID
        assert f(lib, g=None) == INVALID
        assert f(lib, er=None) == INVALID                        # sparse entity table without rows
        assert f(lib, de=None) == INVALID
        assert f(lib, lde=8) == INVALID
        assert f(lib, model=5, l_norm=2.0) == INVALID            # TransE L2 needs the forward's z
        assert f(lib, model=5, l_norm=2.0, z=C.addressof((C.c_float * 64)()), ldz=4) == WORKSPACE


@pytest.mark.parametrize("model", [0, 4, 5, 6])
def test_workspace_bytes_grow_with_the_problem(lib, model):
    Dm = 16 if model == 4 else 128

    def bwd(n=512, nu=1001, E_=40943, R_=237):
        return lib.b200kge_ns_shared_backward_workspace_bytes(model, n, nu, Dm, E_, R_)

    def fwd(n=512, nu=1001):
        return lib.b200kge_ns_shared_score_workspace_bytes(model, n, nu, Dm)

    assert bwd() > 0 and fwd() > 0
    assert bwd(n=1024) > bwd() and bwd(nu=2001) > bwd() and bwd(E_=4_800_000) > bwd()
    assert fwd(n=1024) > fwd() and fwd(nu=2001) > fwd()
    assert bwd(n=-1) == 0 and fwd(nu=-1) == 0


# ---- the job on the CPU (engine stand-ins)
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
    ns_shared_score / ns_shared_backward over the mirrored column map; counts the calls."""
    import engine_stub
    import ns_sparse_oracle as nsp
    from kge_b200 import engine

    calls = {"ns_loss": 0, "ns_backward": 0, "ns_backward_sparse": 0, "shared_score": 0, "shared_backward": 0,
             "shared_sparse": [], "impl": set()}
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

    def negatives(triples, unique, repeat, drop, K):
        n = triples.shape[0]
        U = unique.numel() - (1 if drop is not None else 0)
        rp = repeat.long().reshape(-1).numpy() if repeat is not None else np.zeros(0, np.int64)
        return unique[torch.from_numpy(u_map(n, K, U, rp, None if drop is None else drop.numpy()))]

    def ns_shared_score(model, ent, rel, triples, slot, unique, repeat, drop, K, l_norm=1.0, precision="auto",
                        implementation="batch", want_z=False):
        calls["shared_score"] += 1
        calls["impl"].add(implementation)
        block = engine_stub.ns_score(model, ent, rel, triples, negatives(triples, unique, repeat, drop, K), slot, True,
                                     l_norm)
        if not want_z:
            return block
        un = unique.reshape(1, -1).expand(triples.shape[0], -1)
        return block, engine_stub.ns_score(model, ent, rel, triples, un, slot, False, l_norm)

    def ns_shared_backward(model, ent, rel, triples, slot, unique, repeat, drop, K, grad_scores, z=None, l_norm=1.0,
                           implementation="batch", sparse=(False, False)):
        calls["shared_backward"] += 1
        calls["shared_sparse"].append(tuple(sparse))
        neg = negatives(triples, unique, repeat, drop, K)
        d_ent, d_rel = _dense_grads(model, ent, rel, triples, slot, neg, grad_scores, l_norm)
        tri = triples.long()
        shared = unique if implementation == "batch" else neg.reshape(-1)
        rows_e = (torch.arange(ent.shape[0]) if implementation == "all"
                  else torch.unique(torch.cat((tri[:, 0], tri[:, 2], shared))))
        rows_r = torch.unique(tri[:, 1])
        return (_as_sparse(d_ent, rows_e) if sparse[0] else d_ent, _as_sparse(d_rel, rows_r) if sparse[1] else d_rel)

    names = ("ns_loss", "ns_backward", "ns_backward_sparse", "ns_shared_score", "ns_shared_backward")
    with engine_stub.installed():
        saved = {k: getattr(engine, k) for k in names}
        for k, f in zip(names, (ns_loss, ns_backward, ns_backward_sparse, ns_shared_score, ns_shared_backward)):
            setattr(engine, k, f)
        try:
            yield calls
        finally:
            for k, v in saved.items():
                setattr(engine, k, v)


def _extra(option, shared_type="default", replacement=True, impl="batch", **more):
    extra = {"negative_sampling.num_samples.s": 5, "negative_sampling.num_samples.o": 7,
             "negative_sampling.shared": True, "negative_sampling.shared_type": shared_type,
             "negative_sampling.with_replacement": replacement, "negative_sampling.implementation": impl,
             "train.loss_arg": 0.5}
    if option:
        extra["user.b200_ns_shared"] = True
    extra.update(more)
    return extra


def _train_pair(splits, extra, model="complex", loss="kl", mutate=None, batch_size=16):
    """Two epochs of the plugin job (`extra` as given) and of the reference job (without the user.* options) from the
    same tables and seeds, so both draw the same shared samples; keys starting with "M." are the model's options."""
    import jobs_util as ju

    def cfg(tag):
        name = model if tag == "ref" else "b200_" + model
        return {k.replace("M.", name + ".", 1): v for k, v in extra.items()
                if not (tag == "ref" and k.startswith("user."))}

    torch.manual_seed(0)
    init = ju.make_job(model, E, R, D, splits, train_type="negative_sampling", loss=loss, batch_size=batch_size,
                       extra=cfg("ref"))
    out = {}
    for tag in ("ref", "plugin"):
        kw = {"job_class": "B200TrainingJobNegativeSampling"} if tag == "plugin" else {}
        job = ju.make_job(model if tag == "ref" else "b200_" + model, E, R, D, splits, train_type="negative_sampling",
                          loss=loss, batch_size=batch_size, forward_only=False, extra=cfg(tag), **kw)
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
@pytest.mark.parametrize("shared_type,replacement", [("default", True), ("default", False), ("naive", True),
                                                     ("naive", False)])
def test_option_on_trains_the_shared_slots_natively(splits, stub, shared_type, replacement, loss):
    out = _train_pair(splits, _extra(True, shared_type, replacement), loss=loss)
    assert stub["shared_backward"] > 0 and stub["ns_backward"] == 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


@pytest.mark.parametrize("shared_type", ["default", "naive"])
def test_option_on_with_sub_batches(splits, stub, shared_type):
    out = _train_pair(splits, _extra(True, shared_type, **{"train.subbatch_size": 5}))
    assert stub["shared_backward"] > 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


@pytest.mark.parametrize("model,more", [("transe", {"M.l_norm": 1.0}), ("transe", {"M.l_norm": 2.0}),
                                        ("rotate", {})])
@pytest.mark.parametrize("impl", ["triple", "batch"])
def test_distance_models_pass_the_implementation(splits, stub, model, more, impl):
    # against the option-off plugin job: the stand-ins' TransE L1 differs from the reference's cdist / pairwise_distance
    # by 1.5e-4 on either route
    off = _train_pair(splits, _extra(False, impl=impl, **more), model=model)
    out = _train_pair(splits, _extra(True, impl=impl, **more), model=model)
    assert stub["shared_backward"] > 0 and stub["impl"] == {impl}, stub
    assert out["plugin"] == pytest.approx(off["plugin"], rel=1e-6)


@pytest.mark.parametrize("impl", ["triple", "batch", "all"])
@pytest.mark.parametrize("sparse_ent,sparse_rel", [(True, True), (True, False), (False, True)])
def test_sparse_tables_take_the_row_sparse_output(splits, stub, impl, sparse_ent, sparse_rel):
    more = {"M.entity_embedder.sparse": sparse_ent, "M.relation_embedder.sparse": sparse_rel,
            "train.optimizer.default.type": "Adagrad"}
    out = _train_pair(splits, _extra(True, impl=impl, **more))
    assert stub["shared_backward"] > 0, stub
    assert set(stub["shared_sparse"]) == {(sparse_ent, sparse_rel)}
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_reciprocal_wrapper_s_slot_uses_the_o_slot_form(splits, stub):
    import jobs_util as ju

    extra = _extra(True)
    extra["reciprocal_relations_model.base_model.type"] = "b200_complex"
    out = {}
    for tag, job_class in (("ref", None), ("plugin", "B200TrainingJobNegativeSampling")):
        e = dict(extra)
        if tag == "ref":
            e.pop("user.b200_ns_shared")
            e["reciprocal_relations_model.base_model.type"] = "complex"
        torch.manual_seed(0)
        job = ju.make_job("reciprocal_relations_model", E, R, D, splits, train_type="negative_sampling", loss="kl",
                          batch_size=16, forward_only=False, extra=e, imports=("b200_complex", "complex"),
                          **({"job_class": job_class} if job_class else {}))
        job.epoch += 1
        job._prepare()
        ju.seed_all(10)
        out[tag] = job.run_epoch()["avg_loss"]
    assert stub["shared_backward"] > 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_option_off_changes_nothing(splits, stub):
    out = _train_pair(splits, _extra(False))
    assert stub["shared_score"] == 0 and stub["shared_backward"] == 0 and stub["ns_backward"] > 0, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def _not_shared(stub):
    assert stub["shared_score"] == 0 and stub["shared_backward"] == 0, stub


def test_dropout_falls_through(splits, stub):
    more = {"M.entity_embedder.dropout": 0.2, "M.relation_embedder.dropout": 0.1}
    out = _train_pair(splits, _extra(True, **more))
    _not_shared(stub)
    assert len(out["plugin"]) == 2


def test_p_slot_falls_through(splits, stub):
    out = _train_pair(splits, _extra(True, **{"negative_sampling.num_samples.p": 3}))
    _not_shared(stub)
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_not_shared_sampling_falls_through(splits, stub):
    out = _train_pair(splits, _extra(True, **{"negative_sampling.shared": False}))
    _not_shared(stub)
    assert stub["ns_backward"] > 0
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


def test_frequency_sampling_falls_through(splits, stub):
    import jobs_util as ju

    # shared frequency sampling is not offered by the reference (KgeSampler._sample_shared raises)
    extra = _extra(True, **{"negative_sampling.sampling_type": "frequency"})
    with pytest.raises(Exception):
        job = ju.make_job("b200_complex", E, R, D, splits, train_type="negative_sampling", loss="kl", batch_size=16,
                          forward_only=False, extra=extra, job_class="B200TrainingJobNegativeSampling")
        job.epoch += 1
        job._prepare()
        job.run_epoch()
    _not_shared(stub)


def test_non_b200_model_falls_through(splits, stub):
    import jobs_util as ju

    job = ju.make_job("complex", E, R, D, splits, train_type="negative_sampling", loss="kl", batch_size=16,
                      forward_only=False, extra=_extra(True), job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    job._prepare()
    ju.seed_all(10)
    assert job.run_epoch()["avg_loss"] > 0
    _not_shared(stub)


def test_unserved_norm_falls_through(splits, stub):
    out = _train_pair(splits, _extra(True, **{"M.l_norm": 3.0}), model="transe")
    _not_shared(stub)
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)


@pytest.mark.parametrize("option", [False, True])
def test_naive_sub_batches_train(splits, stub, option):
    # NaiveSharedNegativeSample.samples(slice) raises TypeError (len of a slice); the job slices samples() instead
    out = _train_pair(splits, _extra(option, "naive", **{"train.subbatch_size": 5}))
    assert (stub["shared_backward"] > 0) == option, stub
    assert out["plugin"] == pytest.approx(out["ref"], rel=1e-5)
