"""KvsAll's s_o query type (relation prediction) on the H100: b200kge_score_so_loss_csr and its backward (loss, row
losses, d_ent, d_rel) against fp64 autograd of the reference's generic s_o expression (kge_model.py:202-209) on the
densified labels, with and without embedding dropout, the masks of streams 24-26 against the CPU mirror, and
B200TrainingJobKvsAll training sp_ + s_o + _po against the unmodified job and the CPU reference."""
import pytest
import torch

from kge_b200 import hostenv

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")

TOL = 1e-4          # of the fp64 value's rms (DESIGN §5)
# RESCAL beyond D = 32 (K = D^2 > 1024) does NOT meet the 1e-4 bar: the CUDA-core scorer recomputes each score as one
# fp32 reduction of length K (16384 at D = 128), and with kl the gradients reach 4.3e-4 (5.7e-4 under dropout) of the
# fp64 rms in d_rel on an H100 (DESIGN §9).  Those shapes are held to 1e-3 so that a further loss of precision fails.
TOL_LONG_K = 1e-3
MODELS = ["complex", "distmult", "simple", "cp", "rescal"]
P_ENT, P_REL = 0.4, 0.2
SO_S, SO_O, SO_TABLE = 24, 25, 26


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


def _close(got, ref, what, tol=TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-12)
    err = float((got - ref).abs().max())
    assert err <= tol * rms, f"{what}: max|d| = {err:.3e} > {tol} * rms {rms:.3e}"


def _problem(model, E, R, D, n, seed):
    """Tables, pairs and sorted CSR relation labels: row 0 repeats a label, row 1 has a single label."""
    from oracle import kge_oracle as orc

    g = torch.Generator().manual_seed(seed)
    ent = torch.randn(E, D, generator=g) * 0.3
    rel = torch.randn(R, orc.relation_dim(model, D), generator=g) * 0.3
    s, o = torch.randint(0, E, (n,), generator=g), torch.randint(0, E, (n,), generator=g)
    rows = []
    for i in range(n):
        if i == 0:
            rows.append(torch.tensor([1, 1, R - 1]))
        elif i == 1:
            rows.append(torch.tensor([2]))
        else:
            k = int(torch.randint(1, min(R, 6) + 1, (1,), generator=g))
            rows.append(torch.randperm(R, generator=g)[:k].sort().values)
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.tensor([len(r) for r in rows]), 0)
    return ent, rel, s, o, offs, torch.cat(rows).long()


def _masks(eng, key, n, E, D, R, Dr):
    """(s rows, o rows, relation table) keep masks of the three s_o draws from the library, as float64 multipliers."""
    from dropout_oracle import scale

    def m(p, stream, rows, dim, base):
        return eng.dropout_mask(p, key.seed, key.call, stream, rows, dim, base).double() * scale(p)

    return (m(key.p_ent, SO_S, n, D, key.row_base), m(key.p_ent, SO_O, n, D, key.row_base),
            m(key.p_rel, SO_TABLE, R, Dr, 0))


def _ref_rows(model, ent, rel, s, o, offs, cols, loss, offset, masks=None):
    """Per-row fp64 losses of score_so through the generic s_o expansion, row-chunked to bound its [n R, K] operands."""
    import so_oracle as so
    from oracle import kge_oracle as orc

    se, oe, r = ent[s], ent[o], rel
    if masks is not None:
        se, oe, r = se * masks[0], oe * masks[1], r * masks[2]
    n, R = s.numel(), rel.shape[0]
    chunk = max(1, int(2 ** 27 // max(1, R * rel.shape[1])))
    x = torch.cat([orc.score_emb(model, se[i:i + chunk], r, oe[i:i + chunk], "s_o") for i in range(0, n, chunk)])
    y = so.csr_labels(offs, cols, n, R, torch.float64).to(x.device)
    if loss == "bce":
        z = x + offset
        return (torch.nn.functional.softplus(z) - y * z).sum(1)
    yn = y / y.sum(1, keepdim=True).clamp_min(1e-12)
    lp = torch.log_softmax(x, 1)
    return torch.where(yn > 0, yn * (torch.log(yn.clamp_min(1e-300)) - lp), torch.zeros_like(yn)).sum(1)


SHAPES = {"toy": (11, 5, 16, 7), "multi-tile": (5003, 237, 128, 600), "bench": (14541, 237, 512, 1024),
          "rescal64": (500, 237, 64, 64), "rescal128": (500, 237, 128, 64)}


def _cases():
    out = []
    for shape in SHAPES:
        models = MODELS
        if shape in ("multi-tile",):
            models = [m for m in MODELS if m != "rescal"]
        elif shape == "bench":
            models = ["complex", "distmult"]
        elif shape.startswith("rescal"):
            models = ["rescal"]
        for model in models:
            for loss in ("bce", "kl"):
                for drop in (False, True):
                    for prec in (("auto",) if shape == "bench" else ("auto", "fp32")):
                        out.append((shape, model, loss, drop, prec))
    return out


@pytest.mark.parametrize("shape,model,loss,drop,prec", _cases(), ids=lambda v: str(v))
def test_loss_and_gradients_against_fp64(eng, shape, model, loss, drop, prec):
    E, R, D, n = SHAPES[shape]
    ent, rel, s, o, offs, cols = _problem(model, E, R, D, n, seed=17 * len(shape) + MODELS.index(model))
    dev = "cuda"
    ent_d, rel_d, s_d, o_d, offs_d, cols_d = (t.to(dev) for t in (ent, rel, s, o, offs, cols))
    offset = 0.5 if loss == "bce" else 0.0
    key = eng.DropoutKey(P_ENT, P_REL, 1234, 77, 40) if drop else None
    bs = n + 3
    val, rows = eng.score_so_loss_csr(model, ent_d, rel_d, s_d, o_d, offs_d, cols_d, loss, offset, prec,
                                      return_rows=True, dropout=key)
    d_ent, d_rel = eng.score_so_loss_csr_backward(model, ent_d, rel_d, s_d, o_d, offs_d, cols_d, loss, offset, bs,
                                                  dropout=key)
    masks = _masks(eng, key, n, E, D, R, rel.shape[1]) if drop else None
    e64 = ent_d.double().requires_grad_(True)
    r64 = rel_d.double().requires_grad_(True)
    ref_rows = _ref_rows(model, e64, r64, s_d, o_d, offs_d, cols_d, loss, offset, masks)
    total = ref_rows.sum()
    de, dr = torch.autograd.grad(total / bs, (e64, r64))
    assert float(val) == pytest.approx(float(total.detach()), rel=1e-5, abs=1e-4)
    tol = TOL if rel.shape[1] <= 1024 else TOL_LONG_K
    _close(rows.view(-1, 1), ref_rows.detach().view(-1, 1), "row losses", tol)
    # d_ent is nonzero on the pairs' entity rows only: those rows are held to the rms of their fp64 value (the whole
    # table's rms would shrink the bar by sqrt(E / #rows)), every other row must be exactly zero
    support = torch.unique(torch.cat((s, o)))
    off = torch.ones(E, dtype=torch.bool)
    off[support] = False
    assert not d_ent.cpu()[off].any()
    _close(d_ent.cpu()[support], de.cpu()[support], "d_ent", tol)
    _close(d_rel, dr, "d_rel", tol)


@pytest.mark.parametrize("stream,rows,dim,base", [(SO_S, 7, 16, 40), (SO_O, 9, 24, 3), (SO_TABLE, 237, 16, 0)])
def test_so_masks_match_the_mirror(eng, stream, rows, dim, base):
    """The masks of streams 24-26 bit for bit against the CPU Philox mirror."""
    import dropout_oracle as do

    got = eng.dropout_mask(0.4, 99, 5, stream, rows, dim, base).bool().cpu()
    assert torch.equal(got, do.mask(0.4, 99, 5, stream, rows, dim, base))


def test_distance_family_is_refused(eng):
    ent, rel = torch.randn(10, 8, device="cuda"), torch.randn(3, 8, device="cuda")
    idx, offs, cols = (torch.zeros(2, dtype=torch.int64, device="cuda"), torch.tensor([0, 1, 2], device="cuda"),
                       torch.zeros(2, dtype=torch.int64, device="cuda"))
    with pytest.raises(NotImplementedError):
        eng.score_so_loss_csr("transe", ent, rel, idx, idx, offs, cols)


# ---- training jobs ---------------------------------------------------------------------------------------------------
JE, JR, JD = 200, 12, 32
QTYPES = {"KvsAll.query_types.sp_": True, "KvsAll.query_types.s_o": True, "KvsAll.query_types._po": True}


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(JE, JR, 600, 60, 60)


@pytest.fixture()
def so_calls(eng, monkeypatch):
    calls = []
    orig = eng.score_so_loss_csr_backward

    def counted(*a, **kw):
        calls.append(kw.get("dropout"))
        return orig(*a, **kw)

    monkeypatch.setattr(eng, "score_so_loss_csr_backward", counted)
    return calls


def _run(job, init):
    import jobs_util as ju

    ju.copy_tables(init, job)
    out = []
    for ep in range(2):
        job.epoch += 1
        if job.loader is None:
            job._prepare()
        ju.seed_all(10 + ep)
        out.append(job.run_epoch()["avg_loss"])
    return out


def _cfg(name, dropout, eps):
    c = dict(QTYPES, **{"KvsAll.label_smoothing": eps})
    if dropout:
        c.update({f"{name}.entity_embedder.dropout": P_ENT, f"{name}.relation_embedder.dropout": P_REL})
    return c


def _job(name, splits, loss, cfg, device, job_class=None):
    import jobs_util as ju

    return ju.make_job(name, JE, JR, JD, splits, device=device, train_type="KvsAll", loss=loss, batch_size=64,
                       forward_only=False, extra=cfg, job_class=job_class)


def _assert_tracks(got, ref):
    assert got[0] == pytest.approx(ref[0], rel=1e-4)
    assert got[1] == pytest.approx(ref[1], rel=1e-3)


@needs_ref
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("model", MODELS)
def test_job_against_the_cpu_reference(eng, model, dropout, splits, so_calls):
    """Two epochs (forward, backward, Adagrad) of B200TrainingJobKvsAll with sp_ + s_o + _po track the unmodified job
    on the CPU reference (the mirror's masks patched in under dropout)."""
    import so_oracle as so
    import jobs_util as ju

    loss, eps = ("kl", 0.1) if model in ("complex", "rescal") else ("bce", 0.0)
    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, train_type="KvsAll", loss=loss, batch_size=64,
                       extra=_cfg(model, dropout, eps))
    ref = _job(model, splits, loss, _cfg(model, dropout, eps), "cpu")
    if dropout:
        so.patch_reference_job(ref, P_ENT, P_REL)
    ref_losses = _run(ref, init)
    b200 = _job("b200_" + model, splits, loss, _cfg("b200_" + model, dropout, eps), "cuda", "B200TrainingJobKvsAll")
    _assert_tracks(_run(b200, init), ref_losses)
    assert so_calls and all((k is not None) == dropout for k in so_calls)


@needs_ref
@pytest.mark.parametrize("model", MODELS)
def test_job_against_the_unmodified_job_on_the_plugin_model(eng, model, splits, so_calls):
    """The same plugin model trained by the unmodified TrainingJobKvsAll (s_o through the generic expansion and dense
    labels) and by B200TrainingJobKvsAll (s_o through the new entries)."""
    import jobs_util as ju

    name = "b200_" + model
    torch.manual_seed(0)
    init = ju.make_job(model, JE, JR, JD, splits, train_type="KvsAll", loss="kl", batch_size=64,
                       extra=_cfg(model, False, 0.0))
    plain = _run(_job(name, splits, "kl", _cfg(name, False, 0.0), "cuda"), init)
    assert not so_calls
    fused = _run(_job(name, splits, "kl", _cfg(name, False, 0.0), "cuda", "B200TrainingJobKvsAll"), init)
    assert so_calls
    _assert_tracks(fused, plain)
