"""KvsAll with CSR labels for the distance family on the H100: the backward entries (plain and under embedding dropout)
against fp64 autograd of the reference expression on the densified labels, the forward with label smoothing (whose row
score sums come from the CUDA-core scoring pass), the refusals of uncovered norms, and B200TrainingJobKvsAll training
TransE and RotatE natively against the reference job."""
import pytest
import torch

from kge_b200 import hostenv

pytestmark = pytest.mark.gpu

TOL = 1e-4          # of the reference gradient's rms, as tests/test_gpu_backward.py
CASES = [("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)]
# (streams of the query rows, relation rows, table) of the sp_ and _po query types (include/b200kge.h)
STREAMS = {"sp_": (0, 1, 2), "_po": (5, 4, 3)}


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


def _close(got, ref, what, tol=TOL, bounds=None):
    """max|d| <= tol * rms; bounds (row -> per-element fp64 bound) adds tol * bound to the allowance of a row whose
    gradient sums many terms: each element's sum of |contributions|, which is what its fp32 error scales with."""
    got, ref = got.double().cpu(), ref.double().cpu()
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    allowed = torch.full_like(ref, tol * rms)
    for row, b in (bounds or {}).items():
        allowed[row] += tol * b.double().cpu()
    ratio = (got - ref).abs() / allowed
    i, k = divmod(int(ratio.argmax()), ref.shape[1])
    assert float(ratio[i, k]) <= 1.0, \
        f"{what}: [{i}, {k}] |d|={float((got - ref)[i, k].abs()):.3e} allowed={float(allowed[i, k]):.3e} rms={rms:.3e}"


def _tables(model, E, R, D, n, seed):
    from oracle import kge_oracle as orc

    g = torch.Generator().manual_seed(seed)
    ent = torch.randn(E, D, generator=g) * 0.3
    rel = torch.randn(R, orc.relation_dim(model, D), generator=g) * 0.3
    q, p = torch.randint(0, E, (n,), generator=g), torch.randint(0, R, (n,), generator=g)
    return ent, rel, q, p


def _csr(n, E, seed):
    """Sorted CSR labels with repeated columns, one row listing every column and one row without labels."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for i in range(n):
        if i == 3:
            rows.append(torch.arange(E))
        elif i == 7:
            rows.append(torch.zeros(0, dtype=torch.int64))
        else:
            c = torch.randint(1, 6, (1,), generator=g).item()
            cols = torch.randint(0, E, (c,), generator=g)
            if i % 5 == 1:
                cols = torch.cat((cols, cols[:2]))          # duplicates add up
            rows.append(torch.sort(cols)[0])
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.tensor([len(r) for r in rows]), 0)
    return offs, torch.cat(rows)


class _ModulusL1(torch.autograd.Function):
    """-sum_k |q_k - t_k| over complex elements with the kernels' gradient 0 at |q_k - t_k| = 0, where the reference
    expression's sqrt gives NaN; dropout makes such ties common."""

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


def _score(model, a, r, t, combine, l_norm):
    from oracle import kge_oracle as orc

    if model == "transe":
        # transe.py: -cdist(s + p, o) | -cdist(o - p, s).  The kernels fold in fp32; the fold takes that rounding here
        # too (its gradient is the identity), so L1's sign(q - t) agrees with theirs at near-ties
        q = a + r if combine == "sp_" else a - r
        q32 = (a.float() + r.float()) if combine == "sp_" else (a.float() - r.float())
        q = q + (q32.double() - q).detach()
        return -torch.cdist(q, t, p=l_norm, compute_mode="donot_use_mm_for_euclid_dist")
    if model == "rotate" and l_norm == 1.0:
        h = a.shape[1] // 2
        c, sn = torch.cos(r), torch.sin(r)
        a_re, a_im = a[:, :h], a[:, h:]
        if combine == "sp_":
            q = torch.cat((a_re * c - a_im * sn, a_re * sn + a_im * c), 1)
        else:
            q = torch.cat((c * a_re + sn * a_im, c * a_im - sn * a_re), 1)
        return _ModulusL1.apply(q, t)
    return orc.score_emb(model, a, r, t, "sp_", l_norm) if combine == "sp_" else \
        orc.score_emb(model, t, r, a, "_po", l_norm)


def _ref_loss(model, combine, ent, rel, q, p, offs, cols, loss, offset, eps, l_norm, masks=None):
    """Sum over rows of the KvsAll loss of one query type (the reference expression on dense labels), optionally on
    masked operands masks = (query-row mask, relation-row mask, table mask)."""
    from oracle import kge_oracle as orc

    a, r, t = ent[q], rel[p], ent
    if masks is not None:         # the kernels' masked copies are fp32: same rounding here, identity gradient
        a, r, t = (x * m + ((x * m).float().double() - x * m).detach() for x, m in zip((a, r, t), masks))
    x = _score(model, a, r, t, combine, l_norm)
    n, m = x.shape
    y = torch.zeros((n, m), dtype=x.dtype, device=x.device)
    counts = offs[1:] - offs[:-1]
    y.index_put_((torch.repeat_interleave(torch.arange(n), counts).to(x.device), cols.to(x.device)),
                 torch.ones(len(cols), dtype=x.dtype, device=x.device), accumulate=True)
    if eps > 0:
        y = orc.kvsall_smooth_labels(y, eps)
    return orc.bce_loss(x, y, offset) if loss == "bce" else orc.kl_loss(x, y)


def _grads(fn, ent, rel):
    """fp64 autograd of fn, on the GPU (the multi-tile shapes' [n, E, D] intermediates)."""
    e, r = ent.double().cuda().requires_grad_(True), rel.double().cuda().requires_grad_(True)
    with torch.enable_grad():
        val = fn(e, r)
        de, dr = torch.autograd.grad(val, (e, r))
    return val.detach(), de, dr


def _isolate_dense_row(q, p, E, lo, hi):
    """Row 3 lists every column: give it a query entity and a relation (from [lo, hi)) that no other row uses, so the
    rows of d_ent / d_rel that sum its E terms hold nothing else."""
    p = lo + (p - lo) % (hi - lo - 1)
    p[3] = hi - 1
    q = q.clone()
    q[3] = min(set(range(E)) - set(q[torch.arange(len(q)) != 3].tolist()))
    return q, p


def _dense_row_bounds(model, combine, l_norm, a, r, t, loss, offset, eps, bs):
    """Per element of the query entity row a [D] and relation row r [Dr] of the every-column row (fp64, masked operands
    when dropout is on): sum_j |dL/dz_j * dz_j/d(element)|, the sum of absolute contributions over the E columns."""
    E = t.shape[0]
    with torch.no_grad():
        z = _score(model, a[None], r[None], t, combine, l_norm)[0]
        y = torch.full_like(z, (1.0 - eps) + (1.0 / E if eps > 0 else 0.0))
        g = (torch.sigmoid(z + offset) - y if loss == "bce" else torch.softmax(z, 0) - y / y.sum()).abs() / bs
        if model == "transe":
            q = a + r if combine == "sp_" else a - r
            d = q[None] - t
            w = torch.ones_like(d) if l_norm == 1.0 else d.abs() / d.norm(dim=1, keepdim=True)
            b = (g[:, None] * w).sum(0)
            return b, b
        h = a.shape[0] // 2
        c, sn = torch.cos(r), torch.sin(r)
        if combine == "sp_":
            q_re, q_im = a[:h] * c - a[h:] * sn, a[:h] * sn + a[h:] * c
        else:
            q_re, q_im = c * a[:h] + sn * a[h:], c * a[h:] - sn * a[:h]
        d_re, d_im = q_re[None] - t[:, :h], q_im[None] - t[:, h:]
        mod = torch.sqrt(d_re * d_re + d_im * d_im).clamp_min(1e-300)
        u_re, u_im = (d_re / mod).abs(), (d_im / mod).abs()
        g = g[:, None]
        c, sn = c.abs(), sn.abs()
        b_a = torch.cat(((g * (u_re * c + u_im * sn)).sum(0), (g * (u_re * sn + u_im * c)).sum(0)))
        b_r = (g * (u_re * q_im.abs() + u_im * q_re.abs())).sum(0)
        return b_a, b_r


# ---- 1. the backward entry ------------------------------------------------------------------------------------------
SHAPES = {"ragged": (1201, 11, 48, 90), "multi_tile": (5003, 13, 64, 600)}     # E, R, D, n


def _backward_cases():
    out = []
    for model, l_norm in CASES:
        for combine in ("sp_", "_po"):
            for loss, eps in (("bce", 0.0), ("bce", 0.1), ("kl", 0.0), ("kl", 0.1)):
                out.append((model, l_norm, combine, loss, eps, "ragged"))
            out.append((model, l_norm, combine, "kl", 0.1, "multi_tile"))
            out.append((model, l_norm, combine, "bce", 0.0, "multi_tile"))
    return out


@pytest.mark.parametrize("model,l_norm,combine,loss,eps,shape", _backward_cases())
def test_backward_entry_against_fp64(eng, model, l_norm, combine, loss, eps, shape):
    E, R, D, n = SHAPES[shape]
    ent, rel, q, p = _tables(model, E, R, D, n, seed=11)
    q, p = _isolate_dense_row(q, p, E, 0, R)
    offs, cols = _csr(n, E, seed=12)
    offset = 0.5 if loss == "bce" else 0.0
    bs = 2 * n
    val, de, dr = _grads(lambda e, r: _ref_loss(model, combine, e, r, q, p, offs, cols, loss, offset, eps, l_norm) / bs,
                         ent, rel)
    ec, rc = ent.cuda(), rel.cuda()
    qc, pc, oc, cc = q.cuda(), p.cuda(), offs.cuda(), cols.cuda()
    got = eng.score_1vsN_loss_csr(model, combine, ec, rc, ec, oc, cc, qc, pc, loss, offset, eps, l_norm) / bs
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.score_1vsN_loss_csr_backward(model, combine, ec, rc, qc, pc, oc, cc, loss, offset, eps, bs,
                                              l_norm=l_norm)
    e64, r64 = ent.double(), rel.double()
    b_a, b_r = _dense_row_bounds(model, combine, l_norm, e64[q[3]], r64[p[3]], e64, loss, offset, eps, bs)
    _close(ge, de, "d_ent", bounds={int(q[3]): b_a})
    _close(gr, dr, "d_rel", bounds={int(p[3]): b_r})


# ---- 2. the forward with label smoothing -----------------------------------------------------------------------------
@pytest.mark.parametrize("combine", ["sp_", "_po"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,l_norm", CASES + [("transe", 3.0), ("rotate", 2.0)])
def test_forward_with_label_smoothing(eng, model, l_norm, loss, combine):
    E, R, D, n = 1201, 11, 48, 300          # 300 rows: three row tiles of the CUDA-core scorer
    ent, rel, q, p = _tables(model, E, R, D, n, seed=21)
    offs, cols = _csr(n, E, seed=22)
    offset = 0.5 if loss == "bce" else 0.0
    e, r = ent.double().cuda(), rel.double().cuda()
    rows = torch.stack([_ref_loss(model, combine, e, r, q[i:i + 1], p[i:i + 1], offs[i:i + 2] - offs[i],
                                  cols[offs[i]:offs[i + 1]], loss, offset, 0.1, l_norm) for i in range(n)])
    ec, rc = ent.cuda(), rel.cuda()
    got, got_rows = eng.score_1vsN_loss_csr(model, combine, ec, rc, ec, offs.cuda(), cols.cuda(), q.cuda(), p.cuda(),
                                            loss, offset, 0.1, l_norm, return_rows=True)
    assert float(got) == pytest.approx(float(rows.sum()), rel=1e-4)
    _close(got_rows[:, None], rows[:, None], "row losses")


# ---- 3. under embedding dropout -------------------------------------------------------------------------------------
def _masks(eng, key, streams, q_rows, r_rows, E, D, Dr):
    """The three draws of a query type as fp64 multipliers: keep mask times the kernels' fp32 scale 1 / (1 - p)."""
    import dropout_oracle as dro

    sq, sr, st = streams
    def draw(p, stream, rows, dim, row_base):
        return eng.dropout_mask(p, key.seed, key.call, stream, rows, dim, row_base).double() * dro.scale(p)

    return (draw(key.p_ent, sq, q_rows, D, key.row_base), draw(key.p_rel, sr, r_rows, Dr, key.row_base),
            draw(key.p_ent, st, E, D, 0))


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("combine,streams", [("sp_", "sp_"), ("_po", "_po"), ("sp_", "_po")])
@pytest.mark.parametrize("model,l_norm", CASES)
def test_dropout_backward_against_fp64(eng, model, l_norm, combine, streams, loss, eps):
    """mask_dir = combine, and the reciprocal _po query type: the sp_ fold of (o, p + R) on the _po streams."""
    E, R, D, n = 1201, 11, 48, 90
    ent, rel, q, p = _tables(model, E, 2 * R, D, n, seed=31)
    q, p = _isolate_dense_row(q, p, E, R, 2 * R) if combine != streams else _isolate_dense_row(q, p, E, 0, 2 * R)
    offs, cols = _csr(n, E, seed=32)
    key = eng.DropoutKey(0.3, 0.2, seed=77, call=9, row_base=40)
    masks = _masks(eng, key, STREAMS[streams], n, n, E, D, rel.shape[1])
    offset = 0.5 if loss == "bce" else 0.0
    bs = 2 * n
    val, de, dr = _grads(lambda e, r: _ref_loss(model, combine, e, r, q, p, offs, cols, loss, offset, eps, l_norm,
                                                masks) / bs, ent, rel)
    ec, rc = ent.cuda(), rel.cuda()
    qc, pc, oc, cc = q.cuda(), p.cuda(), offs.cuda(), cols.cuda()
    got = eng.score_1vsN_loss_csr(model, combine, ec, rc, ec, oc, cc, qc, pc, loss, offset, eps, l_norm, dropout=key,
                                  dropout_streams=streams) / bs
    assert float(got) == pytest.approx(float(val), rel=1e-4)
    ge, gr = eng.score_1vsN_loss_csr_backward(model, combine, ec, rc, qc, pc, oc, cc, loss, offset, eps, bs,
                                              dropout=key, dropout_streams=streams, l_norm=l_norm)
    mq, mr, mt = (m.cpu() for m in masks)
    e64, r64 = ent.double(), rel.double()
    b_a, b_r = _dense_row_bounds(model, combine, l_norm, e64[q[3]] * mq[3], r64[p[3]] * mr[3], e64 * mt, loss, offset,
                                 eps, bs)
    _close(ge, de, "d_ent", bounds={int(q[3]): b_a * mq[3]})
    _close(gr, dr, "d_rel", bounds={int(p[3]): b_r * mr[3]})


# ---- 4. refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("model,l_norm", [("transe", 3.0), ("rotate", 2.0)])
def test_uncovered_norms_are_refused(eng, model, l_norm, dropout):
    E, R, D, n = 301, 5, 32, 20
    ent, rel, q, p = _tables(model, E, R, D, n, seed=41)
    offs, cols = _csr(n, E, seed=42)
    kw = {"dropout": eng.DropoutKey(0.3, 0.2, seed=1, call=2)} if dropout else {}
    with pytest.raises(NotImplementedError):
        eng.score_1vsN_loss_csr_backward(model, "sp_", ent.cuda(), rel.cuda(), q.cuda(), p.cuda(), offs.cuda(),
                                         cols.cuda(), "kl", 0.0, 0.0, n, l_norm=l_norm, **kw)


# ---- 5. the training job ---------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 211, 5, 32


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


@pytest.fixture()
def bwd_calls(eng, monkeypatch):
    """Counts the fused backward calls of the KvsAll job."""
    calls = []
    orig = eng.score_1vsN_loss_csr_backward

    def counted(*a, **kw):
        calls.append(kw.get("l_norm"))
        return orig(*a, **kw)

    monkeypatch.setattr(eng, "score_1vsN_loss_csr_backward", counted)
    return calls


def _force_route(model):
    """Take the CSR-label backward without dropout too (the job takes it under dropout only)."""
    model.b200_kvsall_native_backward_ok = lambda dropout=False: True


def _train_pair(model, l_norm, loss, eps, splits, dropout=False, force_route=False):
    import dropout_oracle as dro
    import jobs_util as ju

    extra = {"KvsAll.label_smoothing": eps}

    def cfg(name):
        c = dict(extra, **{f"{name}.l_norm": l_norm})
        if dropout:
            c.update({f"{name}.entity_embedder.dropout": 0.3, f"{name}.relation_embedder.dropout": 0.1})
        return c

    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, train_type="KvsAll", loss=loss, batch_size=64, extra=cfg(model))
    losses = {}
    for tag in ("ref", "b200"):
        name = model if tag == "ref" else "b200_" + model
        job = ju.make_job(name, JE, JR, JD, splits, device="cpu" if tag == "ref" else "cuda", train_type="KvsAll",
                          loss=loss, batch_size=64, forward_only=False, extra=cfg(name),
                          job_class=None if tag == "ref" else "B200TrainingJobKvsAll")
        if tag == "ref" and dropout:
            dro.patch_reference_job(job, 0.3, 0.1)
        if tag == "b200" and force_route:
            _force_route(job.model)
        ju.copy_tables(init, job)
        out = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            out.append(job.run_epoch()["avg_loss"])
        losses[tag] = out
    return losses


def _assert_tracks(losses):
    assert losses["b200"][0] == pytest.approx(losses["ref"][0], rel=1e-4)
    assert losses["b200"][1] == pytest.approx(losses["ref"][1], rel=1e-3)


@needs_ref
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("loss", ["kl", "bce"])
@pytest.mark.parametrize("model,l_norm", CASES)
def test_kvsall_training_job(eng, model, l_norm, loss, eps, splits, bwd_calls):
    """Two epochs (forward, backward, Adagrad) of B200TrainingJobKvsAll on the CSR-label route track the reference job
    on the CPU."""
    _assert_tracks(_train_pair(model, l_norm, loss, eps, splits, force_route=True))
    assert bwd_calls and all(ln == l_norm for ln in bwd_calls)      # the fused route ran, with the model's norm


@needs_ref
@pytest.mark.parametrize("model,l_norm", CASES)
def test_dropout_free_job_keeps_the_dense_step(eng, model, l_norm, splits, bwd_calls):
    """Without dropout the job keeps the unmodified step (stored dense scores, native dense backward)."""
    _assert_tracks(_train_pair(model, l_norm, "kl", 0.1, splits))
    assert not bwd_calls


@needs_ref
@pytest.mark.parametrize("model,l_norm,loss", [("transe", 1.0, "kl"), ("transe", 2.0, "bce"), ("rotate", 1.0, "kl")])
def test_kvsall_training_job_with_dropout(eng, model, l_norm, loss, splits, bwd_calls):
    """Under embedding dropout, against the reference job drawing the mirror's masks."""
    _assert_tracks(_train_pair(model, l_norm, loss, 0.1, splits, dropout=True))
    assert bwd_calls


@needs_ref
@pytest.mark.parametrize("model,l_norm", [("transe", 3.0), ("rotate", 2.0)])
def test_uncovered_norms_train_through_the_reference_step(eng, model, l_norm, splits, bwd_calls):
    _assert_tracks(_train_pair(model, l_norm, "kl", 0.1, splits))
    assert not bwd_calls


@needs_ref
@pytest.mark.parametrize("dropout", [False, True])
def test_kvsall_training_on_reciprocal_transe(eng, dropout, splits, bwd_calls):
    """reciprocal_relations_model over b200_transe: the _po query type is the sp_ fold of (o, p + R)."""
    import dropout_oracle as dro
    import jobs_util as ju

    def make(bm, dev, cls):
        cfg = {"reciprocal_relations_model.base_model.type": bm, "KvsAll.label_smoothing": 0.1}
        if dropout:
            cfg.update({f"{bm}.entity_embedder.dropout": 0.3, f"{bm}.relation_embedder.dropout": 0.1})
        return ju.make_job("reciprocal_relations_model", JE, JR, JD, splits, device=dev, train_type="KvsAll",
                           loss="kl", batch_size=64, forward_only=False, imports=(bm,), extra=cfg, job_class=cls)

    torch.manual_seed(0)
    init = make("transe", "cpu", None)
    losses = {}
    for tag, dev, bm, cls in (("ref", "cpu", "transe", None), ("b200", "cuda", "b200_transe", "B200TrainingJobKvsAll")):
        job = make(bm, dev, cls)
        if tag == "ref" and dropout:
            dro.patch_reference_job(job, 0.3, 0.1)
        if tag == "b200" and not dropout:
            _force_route(job.model._base_model)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        out = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(20 + ep)
            out.append(job.run_epoch()["avg_loss"])
        losses[tag] = out
    _assert_tracks(losses)
    assert bwd_calls
