"""Embedding dropout on the H100: the mask kernel against the CPU mirror bit for bit, the 1vsAll and KvsAll dropout
entry points (loss, d_ent, d_rel) against fp64 autograd of the masked reference expression with the same masks, the
job plugins against the reference jobs drawing the mirror's masks, determinism, eval mode and the penalty."""
import pytest
import torch

import dropout_oracle as dro
from kge_b200 import hostenv

pytestmark = pytest.mark.gpu

TOL = 1e-4          # of the reference gradient's rms, as tests/test_gpu_backward.py


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


# ---- 1. the mask generator ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("p,seed,call,stream,rows,dim,row_base", [
    (0.3, 0, 0, 0, 7, 37, 0), (0.5, 2 ** 40 + 3, 17, 2, 5, 13, 9), (0.1, 12345, 2 ** 33 + 1, 5, 4, 64, 1000),
    (0.9, 7, 3, 4, 9, 6, 3), (0.0, 1, 1, 1, 3, 5, 0)])
def test_mask_matches_mirror(eng, p, seed, call, stream, rows, dim, row_base):
    got = eng.dropout_mask(p, seed, call, stream, rows, dim, row_base).cpu().bool()
    assert torch.equal(got, dro.mask(p, seed, call, stream, rows, dim, row_base))


def test_mask_refuses_bad_rates(eng):
    with pytest.raises(ValueError):
        eng.dropout_mask(1.0, 0, 0, 0, 4, 4)
    with pytest.raises(ValueError):
        eng.dropout_mask(-0.1, 0, 0, 0, 4, 4)


# ---- 2./3. entry points against fp64 autograd --------------------------------------------------------------------
E, R, D, N = 300, 7, 32, 64
CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
         ("transe", 2.0), ("rotate", 1.0)]


class _ModulusL1(torch.autograd.Function):
    """-sum_k |q_k - t_k| over complex elements with the kernels' convention at |q_k - t_k| = 0: gradient 0, where the
    reference expression's sqrt gives NaN.  Dropout makes such ties common (both halves of a query element and of a
    candidate element dropped); TransE's L1 needs no stand-in, since torch's cdist and the kernel both take sign(0) = 0."""

    @staticmethod
    def forward(ctx, q, t):
        h = q.shape[1] // 2
        dre = q[:, None, :h] - t[None, :, :h]
        dim_ = q[:, None, h:] - t[None, :, h:]
        mod = torch.sqrt(dre * dre + dim_ * dim_)
        ctx.save_for_backward(dre, dim_, mod)
        return -mod.sum(-1)

    @staticmethod
    def backward(ctx, g):
        dre, dim_, mod = ctx.saved_tensors
        inv = torch.where(mod > 0, 1.0 / torch.where(mod > 0, mod, 1.0), 0.0)
        wre, wim = -g.unsqueeze(-1) * dre * inv, -g.unsqueeze(-1) * dim_ * inv
        return torch.cat((wre.sum(1), wim.sum(1)), 1), -torch.cat((wre.sum(0), wim.sum(0)), 1)


def _score(model, q_ent, r, t, combine, l_norm):
    """Scores of one direction; RotatE's L1 uses the kernels' gradient at exact ties (see above)."""
    from oracle import kge_oracle as orc

    if model == "rotate" and l_norm == 1.0:
        h = q_ent.shape[1] // 2
        c, sn = torch.cos(r), torch.sin(r)
        a_re, a_im = q_ent[:, :h], q_ent[:, h:]
        if combine == "sp_":
            q = torch.cat((a_re * c - a_im * sn, a_re * sn + a_im * c), 1)
        else:
            q = torch.cat((c * a_re + sn * a_im, c * a_im - sn * a_re), 1)
        return _ModulusL1.apply(q, t)
    return orc.score_emb(model, q_ent, r, t, combine, l_norm) if combine == "sp_" else \
        orc.score_emb(model, t, r, q_ent, combine, l_norm)


def _ref_1vsall(model, ent, rel, tri, loss, offset, key, l_norm):
    from oracle import kge_oracle as orc

    s, p, o = tri[:, 0], tri[:, 1], tri[:, 2]
    total = 0.0
    for direction, a, lab in ((0, s, o), (1, o, s)):
        sq, sr, st = dro.DIR_STREAMS[direction]
        q = dro.apply(ent[a], key.p_ent, key.seed, key.call, sq, key.row_base)
        r = dro.apply(rel[p], key.p_rel, key.seed, key.call, sr, key.row_base)
        t = dro.apply(ent, key.p_ent, key.seed, key.call, st, 0)
        x = _score(model, q, r, t, "sp_" if direction == 0 else "_po", l_norm)
        total = total + (orc.bce_loss(x, lab, offset) if loss == "bce" else orc.kl_loss(x, lab))
    return total / tri.shape[0]


def _tables(model, seed=0):
    from oracle import kge_oracle as orc

    g = torch.Generator().manual_seed(seed)
    ent = torch.randn(E, D, generator=g) * 0.3
    rel = torch.randn(R, orc.relation_dim(model, D), generator=g) * 0.3
    tri = torch.stack([torch.randint(0, E, (N,), generator=g), torch.randint(0, R, (N,), generator=g),
                       torch.randint(0, E, (N,), generator=g)], 1)
    return ent, rel, tri


@pytest.mark.parametrize("p_rel", [0.0, 0.2])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,l_norm", CASES)
def test_1vsall_dropout_against_fp64(eng, model, l_norm, loss, p_rel):
    ent, rel, tri = _tables(model)
    key = eng.DropoutKey(0.3, p_rel, seed=2024, call=77, row_base=130)
    offset = 0.5 if loss == "bce" else 0.0
    val, de, dr = dro.grads(lambda e, r: _ref_1vsall(model, e, r, tri, loss, offset, key, l_norm),
                            ent.double(), rel.double())
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    got = eng.train_1vsall_forward(model, ec, rc, tc, loss, offset, l_norm, dropout=key)
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.train_1vsall_backward(model, ec, rc, tc, loss, offset, l_norm, dropout=key)
    _close(ge, de, "d_ent")
    _close(gr, dr, "d_rel")


def _csr(n, seed=1):
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(1, 5, (n,), generator=g)
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(counts, 0)
    cols = torch.cat([torch.sort(torch.randint(0, E, (int(c),), generator=g))[0] for c in counts])
    return offs, cols


@pytest.mark.parametrize("eps", [0.0, 0.2])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("combine", ["sp_", "_po"])
@pytest.mark.parametrize("model", ["complex", "distmult", "simple", "cp", "rescal"])
def test_kvsall_dropout_against_fp64(eng, model, combine, loss, eps):
    ent, rel, tri = _tables(model, seed=3)
    q, p = tri[:, 0], tri[:, 1]
    offs, cols = _csr(N)
    key = eng.DropoutKey(0.3, 0.2, seed=99, call=5, row_base=40)
    offset = 0.5 if loss == "bce" else 0.0
    bs = 2 * N
    val, de, dr = dro.grads(lambda e, r: dro.loss_kvsall(model, combine, e, r, q, p, offs, cols, loss, offset, eps, key)
                            / bs, ent.double(), rel.double())
    ec, rc = ent.cuda(), rel.cuda()
    qc, pc, oc, cc = q.cuda(), p.cuda(), offs.cuda(), cols.cuda()
    got = eng.score_1vsN_loss_csr(model, combine, ec, rc, ec, oc, cc, qc, pc, loss, offset, eps, dropout=key) / bs
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.score_1vsN_loss_csr_backward(model, combine, ec, rc, qc, pc, oc, cc, loss, offset, eps, bs, dropout=key)
    _close(ge, de, "d_ent")
    _close(gr, dr, "d_rel")


# ---- 5. same key twice ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["complex", "transe"])
def test_same_key_same_result(eng, model):
    ent, rel, tri = _tables(model, seed=5)
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    key = eng.DropoutKey(0.4, 0.2, seed=1, call=2, row_base=0)
    a = eng.train_1vsall_forward(model, ec, rc, tc, "kl", dropout=key).clone()
    b = eng.train_1vsall_forward(model, ec, rc, tc, "kl", dropout=key)
    assert torch.equal(a, b)
    g1 = eng.train_1vsall_backward(model, ec, rc, tc, "kl", dropout=key)
    g2 = eng.train_1vsall_backward(model, ec, rc, tc, "kl", dropout=key)
    for x, y in zip(g1, g2):                  # the unfold and scatter add with atomics
        _close(x, y, "repeat", tol=1e-6)
    c = eng.train_1vsall_forward(model, ec, rc, tc, "kl", dropout=key._replace(call=3))
    assert not torch.equal(a, c)


# ---- 4./6./7. jobs, eval mode, penalty -----------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 211, 5, 32


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


def _drop_cfg(model, p_ent=0.3, p_rel=0.1):
    return {f"{model}.entity_embedder.dropout": p_ent, f"{model}.relation_embedder.dropout": p_rel}


@needs_ref
@pytest.mark.parametrize("train_type,model,loss", [
    ("1vsAll", "complex", "kl"), ("1vsAll", "cp", "bce"), ("1vsAll", "transe", "kl"), ("1vsAll", "rotate", "bce"),
    ("KvsAll", "complex", "kl"), ("KvsAll", "distmult", "bce")])
def test_training_jobs_with_dropout(eng, train_type, model, loss, splits):
    """Two epochs of the fused job on the GPU against the reference job on the CPU drawing the mirror's masks."""
    import jobs_util as ju

    hostenv.import_kge()
    from kge.model.embedder.lookup_embedder import LookupEmbedder

    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, train_type=train_type, loss=loss, batch_size=64)
    cls = {"1vsAll": "B200TrainingJob1vsAll", "KvsAll": "B200TrainingJobKvsAll"}[train_type]
    losses = {}
    for tag in ("ref", "b200"):
        name = model if tag == "ref" else "b200_" + model
        job = ju.make_job(name, JE, JR, JD, splits, device="cpu" if tag == "ref" else "cuda", train_type=train_type,
                          loss=loss, batch_size=64, forward_only=False, extra=_drop_cfg(name),
                          job_class=None if tag == "ref" else cls)
        if tag == "ref":
            dro.patch_reference_job(job, 0.3, 0.1)
        ju.copy_tables(init, job)
        embed_all_calls = []
        if tag == "b200":
            orig = LookupEmbedder.embed_all
            for emb in (job.model.get_s_embedder(), job.model.get_p_embedder()):
                emb.embed_all = lambda emb=emb: embed_all_calls.append(1) or orig(emb)
        out = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            out.append(job.run_epoch()["avg_loss"])
        losses[tag] = out
        if tag == "b200":
            assert not embed_all_calls                     # the native route ran, not the reference embedders
    assert losses["b200"][0] == pytest.approx(losses["ref"][0], rel=1e-4)
    assert losses["b200"][1] == pytest.approx(losses["ref"][1], rel=1e-3)


@needs_ref
def test_eval_mode_is_the_existing_path(eng, splits):
    import jobs_util as ju

    job = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", loss="kl", batch_size=64,
                      extra=_drop_cfg("b200_complex"))
    model = job.model
    tri = splits["train"][:100].long().cuda()
    model.eval()
    with torch.no_grad():
        a = model.loss_1vsall(tri, "kl", 0.0, need_grad=False).clone()
        e, r = model._b200_tables()
        b = eng.train_1vsall_forward("complex", e, r, tri, "kl", 0.0)
        s1 = model.score_sp(tri[:, 0], tri[:, 1])
        s2 = eng.score_1vsN("complex", "sp_", e, r, e, tri[:, 0], tri[:, 1])
    assert torch.equal(a, b) and torch.equal(s1, s2)


@needs_ref
def test_penalty_with_dropout_runs_the_kernel(eng, splits, monkeypatch):
    import jobs_util as ju

    cfg = dict(_drop_cfg("b200_complex"))
    cfg.update({"b200_complex.entity_embedder.regularize_weight": 0.01, "lookup_embedder.regularize": "lp",
                "b200_complex.relation_embedder.regularize_weight": 0.02})
    job = ju.make_job("b200_complex", JE, JR, JD, splits, device="cuda", loss="kl", batch_size=64, extra=cfg)
    job.model.train()
    emb = job.model.get_s_embedder()
    ran = []
    orig = eng.lookup_penalty
    monkeypatch.setattr(eng, "lookup_penalty", lambda *a, **kw: ran.append(1) or orig(*a, **kw))
    got = emb.penalty()
    ref = type(emb).penalty(emb)
    assert ran and len(got) == len(ref)
    for (_, a), (_, b) in zip(got, ref):
        assert float(a) == pytest.approx(float(b), rel=1e-5)
