"""Every row of the fused BCE and KL losses against the fp64 loss of the kernel's own fp32 scores.

The store form and the fused-loss forms of one batch run the same scoring arithmetic (capi.cu, run_block), so the
scores the loss epilogue saw are read back through score_1vsN / score_sp_po, and each kernel row must lie within the
rounding bound of tests/loss_rows_oracle.py of the fp64 row of those scores.  That isolates the epilogues, the per-row
slots (2 * nsl per row on the tensor-core path, one per column chunk on the CUDA-core and dense paths) and the
finaliser from the scoring error; a label lost on a tile edge, one slot dropped or counted twice, or a wrong neutral
fill moves one row by far more than its bound.  The batch totals are also compared with the fp64 loss of fp64 scores
at the suite's 1e-4 relative bar (not for single-pass tf32, which misses it by design).

Label placement: index labels put, across the rows, the label on columns 0..7 (every residue of the quad's column
pattern 2q + 8j (+1)), 127, 128, 129, 120..127 of the last full tile, and the first and last column of the last tile.
Stress rows: row 1's label column scores 40 above the rest of the row (KL ~ 0), row 2 has a zero query (every score
0: KL = ln E, BCE = E ln(1 + e^off) - off)."""
import pytest
import torch

import loss_rows_oracle as lr
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4
R = 11
ZERO_REL = R - 1         # relation row zeroed: the queries that use it score 0 against every entity
WORST = {}               # mode -> largest |err| / bound seen


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    yield engine
    print("\nlargest |row error| / row bound per mode:")
    for mode, (ratio, what) in sorted(WORST.items()):
        print(f"  {mode:28s} {ratio:.3e}   ({what})")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _edge_cols(E):
    last = 128 * ((E - 1) // 128)
    full = 128 * (E // 128)
    cols = list(range(8)) + [127, 128, 129, last, E - 1] + [c for c in range(full - 8, full) if c >= 0]
    return sorted({c for c in cols if 0 <= c < E})


def _problem(model, E, D, n, sigma=1.0, seed=0, dominant=True):
    """Tables, query rows (s, p) and index labels with the edge placement and the two stress rows."""
    ent, rel = orc.make_tables(model, E, R, D, sigma=sigma)
    if model in orc.GEMM_FAMILY:
        rel[ZERO_REL] = 0.0
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(0, E, (n,), generator=g)
    p = torch.randint(0, R - 1, (n,), generator=g)
    lab = torch.randint(0, E, (n,), generator=g)
    edge = _edge_cols(E)
    for i in range(0, n, 2):
        lab[i] = edge[(i // 2) % len(edge)]
    if n > 2 and model in orc.GEMM_FAMILY:
        p[2] = ZERO_REL
    if n > 1 and dominant and model in orc.GEMM_FAMILY:
        # row 1: its label column E - 1 scores 40 above every other column of the row
        s[1] = 3
        lab[1] = E - 1
        q = orc.score_emb(model, ent[s[1:2]].double(), rel[p[1:2]].double(), torch.eye(D, dtype=torch.float64), "sp_")[0]
        others = orc.score_emb(model, ent[s[1:2]].double(), rel[p[1:2]].double(), ent[:-1].double(), "sp_")
        ent[E - 1] = (q * (float(others.max()) + 40.0) / float(q @ q)).float()
    return ent, rel, s, p, lab


def _check_rows(mode, what, loss, rows, z, labels, depth, offset=0.0, n_log=None, smoothing=0.0, csr=False):
    """Assert |rows_i - fp64_i| <= bound_i for every row; the fp64 rows are of the kernel's own scores z."""
    z = z.double()
    ref = lr.loss_rows(loss, z, labels, offset, smoothing)
    bound = lr.row_bound(loss, z, labels, depth, offset, n_log, smoothing, csr)
    err = (rows.double() - ref).abs()
    ratio = err / bound
    i = int(ratio.argmax())
    r = float(ratio[i])
    if r > WORST.get(mode, (-1.0, ""))[0]:
        WORST[mode] = (r, what)
    assert r <= 1.0, (f"{what}: row {i}: kernel {float(rows[i]):.9g} fp64 {float(ref[i]):.9g} |err| {float(err[i]):.3e}"
                      f" > bound {float(bound[i]):.3e}")
    return ref


def _rel_close(got, ref, what, tol=TOL):
    got, ref = float(got), float(ref)
    assert abs(got - ref) <= tol * abs(ref), f"{what}: {got} vs {ref}"


def _depth(path, loss, nq, m, sms):
    if path == "tc":
        return lr.tc_depth(loss, nq, m, sms, ping_pong=True)
    if path == "tc-split":
        return lr.tc_depth(loss, nq, m, sms, ping_pong=False)
    return lr.simt_depth(loss, nq, m)


def _n_log(path, loss, z, m, offset):
    if loss != "bce":
        return None
    return lr.tc_log_count(z.shape[0], m) if path.startswith("tc") else lr.log_count(z, offset)


def _run_index(eng, sms, model, E, D, n, loss, prec="auto", path="tc", sigma=1.0, offset=0.0, l_norm=1.0,
               mode=None, dominant=True):
    ent, rel, s, p, lab = _problem(model, E, D, n, sigma, dominant=dominant)
    ce, cr, cs, cp = ent.cuda(), rel.cuda(), s.cuda(), p.cuda()
    out, rows = eng.score_1vsN_loss(model, "sp_", ce, cr, ce, lab.cuda(), cs, cp, None, loss, offset, l_norm, prec,
                                    return_rows=True)
    z = eng.score_1vsN(model, "sp_", ce, cr, ce, cs, cp, None, l_norm, prec)
    what = f"{model} E={E} D={D} n={n} {loss} {prec}"
    _check_rows(mode or f"{path} {loss}", what, loss, rows, z, lab.cuda(), _depth(path, loss, n, E, sms), offset,
                _n_log(path, loss, z, E, offset))
    if prec != "tf32":
        zref = orc.score_sp(model, ce.double(), cr.double(), cs, cp, l_norm=l_norm)
        ref = orc.bce_loss(zref, lab.cuda(), offset) if loss == "bce" else orc.kl_loss(zref, lab.cuda())
        _rel_close(out, ref, what)
    return z


# --------------------------------------------------------------------------- the tensor-core schedule
TC_SHAPES = [
    ("complex", 100, 32, 16),        # one tile, the smallest n the auto path sends to the tensor cores
    ("complex", 1000, 256, 100),     # 8 tiles < SMs
    ("distmult", 6007, 512, 389),    # CTA ranges of 2 and 3 tiles straddling query tiles
    ("complex", 3001, 1024, 77),     # 16 K chunks per tile
    ("complex", 1000, 64, 4096),     # n = 4096
    ("complex", 25000, 128, 32),     # one query tile, 196 entity tiles: nsl = 132
    ("distmult", 30000, 256, 64),    # one query tile, 235 entity tiles
    ("distmult", 1024, 128, 200),    # E a multiple of 128
    ("complex", 1025, 128, 129),     # E = 1 (mod 128): a one-column last tile; n = 1 (mod 64)
    ("rescal", 1000, 64, 100),
    ("simple", 1000, 128, 100),
]


@pytest.mark.parametrize("shape", TC_SHAPES, ids=[f"{m}-E{e}-D{d}-n{n}" for m, e, d, n in TC_SHAPES])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_tc_index_label_rows(eng, sms, shape, loss):
    model, E, D, n = shape
    _run_index(eng, sms, model, E, D, n, loss)


@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_tc_f16x3_below_auto_threshold(eng, sms, loss):
    """f16x3 forced for n = 8: one partial query tile, rows 8..127 of the tile absent."""
    _run_index(eng, sms, "complex", 1025, 128, 8, loss, prec="f16x3")


@pytest.mark.parametrize("E", [1024, 1000], ids=["E1024-full", "E1000-ragged"])
@pytest.mark.parametrize("regime", ["far", "near"])
def test_tc_bce_extreme_logit_rows(eng, sms, regime, E):
    """The one-logarithm-per-lane-and-tile BCE form where every factor is 1 (far) or near 2 (near), with an offset."""
    sigma, offset = {"far": (3.0, 0.5), "near": (0.2, 0.1)}[regime]
    _run_index(eng, sms, "complex", E, 256, 389, "bce", sigma=sigma, offset=offset, mode=f"tc bce {regime}",
               dominant=False)


def _multi_hot(n, E, seed, empty_row=None):
    g = torch.Generator().manual_seed(seed)
    dense = (torch.rand((n, E), generator=g) < 0.01).float()
    dense[torch.arange(n), torch.randint(0, E, (n,), generator=g)] = 1.0
    edge = _edge_cols(E)
    for i in range(0, n, 3):
        dense[i, edge[(i // 3) % len(edge)]] = 1.0
    if empty_row is not None:
        dense[empty_row] = 0.0
    return dense


@pytest.mark.parametrize("smoothing", [0.0, 0.1], ids=["multi-hot", "smoothed"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_tc_dense_label_rows(eng, sms, loss, smoothing):
    """Dense labels, one row without label mass (multi-hot) or every entry >= 1/E (smoothed)."""
    model, E, D, n = "complex", 3001, 256, 389
    ent, rel, s, p, _ = _problem(model, E, D, n, sigma=0.5)
    y = _multi_hot(n, E, seed=5, empty_row=4)
    if smoothing:
        y = orc.kvsall_smooth_labels(y, smoothing)
    ce, cr, cs, cp, cy = ent.cuda(), rel.cuda(), s.cuda(), p.cuda(), y.cuda()
    offset = 0.2 if loss == "bce" else 0.0
    out, rows = eng.score_1vsN_loss(model, "sp_", ce, cr, ce, cy, cs, cp, None, loss, offset, return_rows=True)
    z = eng.score_1vsN(model, "sp_", ce, cr, ce, cs, cp)
    what = f"dense labels eps={smoothing} {loss}"
    _check_rows(f"tc {loss} dense", what, loss, rows, z, cy, _depth("tc", loss, n, E, sms), offset,
                _n_log("tc", loss, z, E, offset))
    if smoothing == 0.0 and loss == "kl":
        assert float(rows[4]) == 0.0
    zref = orc.score_sp(model, ce.double(), cr.double(), cs, cp)
    ref = orc.bce_loss(zref, cy.double(), offset) if loss == "bce" else orc.kl_loss(zref, cy.double())
    _rel_close(out, ref, what)


@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_tc_csr_label_rows(eng, sms, loss):
    """CSR labels (score_1vsN_loss_csr): the label-free pass, the listed scores from the same epilogue, one empty row."""
    model, E, D, n = "complex", 3001, 256, 389
    ent, rel, s, p, _ = _problem(model, E, D, n, sigma=0.5)
    y = _multi_hot(n, E, seed=6, empty_row=5)
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = y.sum(1).long().cumsum(0)
    cols = y.nonzero()[:, 1].contiguous()
    ce, cr, cs, cp = ent.cuda(), rel.cuda(), s.cuda(), p.cuda()
    offset = 0.2 if loss == "bce" else 0.0
    out, rows = eng.score_1vsN_loss_csr(model, "sp_", ce, cr, ce, offs.cuda(), cols.cuda(), cs, cp, loss, offset,
                                        return_rows=True)
    z = eng.score_1vsN(model, "sp_", ce, cr, ce, cs, cp)
    depth = _depth("tc", loss, n, E, sms) + lr.csr_extra_depth(offs)
    labels = (offs.cuda(), cols.cuda())
    _check_rows(f"tc {loss} csr", f"CSR labels {loss}", loss, rows, z, labels, depth, offset,
                _n_log("tc", loss, z, E, offset), csr=True)
    zref = orc.score_sp(model, ce.double(), cr.double(), cs, cp)
    yd = lr.dense_labels(labels, n, E)
    ref = orc.bce_loss(zref, yd, offset) if loss == "bce" else orc.kl_loss(zref, yd)
    _rel_close(out, ref, f"CSR labels {loss}")


# --------------------------------------------------------------------------- other slot layouts
@pytest.mark.parametrize("prec,path", [("3xtf32", "tc-split"), ("tf32+bf16x2", "tc-split"), ("tf32", "tc"),
                                       ("fp32", "simt")])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_precision_mode_rows(eng, sms, prec, path, loss):
    """Row-split slots (four warpgroups, h = q >> 1), single-pass tf32 (ping-pong), the CUDA-core column chunks."""
    _run_index(eng, sms, "distmult", 6007, 512, 389, loss, prec=prec, path=path, mode=f"{prec} {loss}")


@pytest.mark.parametrize("model,l_norm", [("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)],
                         ids=["transe-L1", "transe-L2", "rotate-L1"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_distance_model_rows(eng, sms, model, l_norm, loss):
    _run_index(eng, sms, model, 3001, 128, 389, loss, path="simt", sigma=0.1, l_norm=l_norm,
               mode=f"simt {model}-L{int(l_norm)} {loss}")


@pytest.mark.parametrize("labels", ["index", "smoothed"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_loss_dense_rows(eng, loss, labels):
    """loss_dense over stored scores: dense_epilogue_kernel's 4096-column chunks (3 of them) and the finaliser."""
    n, E = 389, 9001
    g = torch.Generator().manual_seed(7)
    z = (torch.randn((n, E), generator=g) * 3.0).cuda()
    if labels == "index":
        lab = torch.randint(0, E, (n,), generator=g)
        lab[: len(_edge_cols(E))] = torch.tensor(_edge_cols(E), dtype=torch.int64)
        lab[5] = 4095
        lab[6] = 4096
        y = lab.cuda()
    else:
        y = orc.kvsall_smooth_labels(_multi_hot(n, E, seed=8), 0.1).cuda()
    offset = -0.3 if loss == "bce" else 0.0
    out, rows = eng.loss_dense(z, y, loss, offset, return_rows=True)
    n_log = lr.log_count(z, offset) if loss == "bce" else None
    ref = _check_rows(f"dense {loss}", f"loss_dense {labels} {loss}", loss, rows, z, y, lr.dense_depth(loss, n, E),
                      offset, n_log)
    _rel_close(out, ref.sum(), f"loss_dense {labels} {loss}")


# --------------------------------------------------------------------------- the fused 1vsAll step
def _step_check(eng, sms, what, loss, got, z, labels, n):
    """The fused step's total against (sum of the fp64 rows of the stacked stored scores) / n.  Bar: the per-row bounds
    plus the finaliser's fixed-order sum of the 2n rows (rows per warp in order, 8 warps, <= 128 block sums: a
    5-level tree) and the 1/n scaling."""
    nq = z.shape[0]
    depth = lr.tc_depth(loss, nq, z.shape[1], sms)
    n_log = lr.tc_log_count(nq, z.shape[1]) if loss == "bce" else None
    ref_rows = lr.loss_rows(loss, z, labels)
    bound = lr.row_bound(loss, z, labels, depth, 0.0, n_log)
    grid = min(128, lr._cdiv(nq, 8))
    d_sum = lr._cdiv(nq, grid * 8) + 8 + lr._cdiv(grid, 32) + 5 + 2
    bar = (float(bound.sum()) + lr.C * lr.U * d_sum * float(ref_rows.abs().sum())) / n
    ref = float(ref_rows.sum()) / n
    err = abs(float(got) - ref)
    mode = f"fused step {loss}"
    if err / bar > WORST.get(mode, (-1.0, ""))[0]:
        WORST[mode] = (err / bar, what)
    assert err <= bar, f"{what}: kernel {float(got):.9g} fp64 of stored scores {ref:.9g} |err| {err:.3e} > bar {bar:.3e}"


def _edge_triples(E, n, seed):
    g = torch.Generator().manual_seed(seed)
    tri = orc.make_triples(E, R - 1, n, seed=seed)
    edge = torch.tensor(_edge_cols(E))
    tri[:, 0] = edge[torch.randint(0, len(edge), (n,), generator=g)]
    tri[:, 2] = edge[torch.randint(0, len(edge), (n,), generator=g)]
    return tri


@pytest.mark.parametrize("case", ["bench-shape", "edge-columns"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_fused_step_total(eng, sms, case, loss):
    """train_1vsall_forward (the step bench.py times) against the stacked score_sp_po scores of the same batch."""
    model, E, D, n = ("complex", 14541, 512, 2048) if case == "bench-shape" else ("complex", 3001, 256, 389)
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.3)
    tri = orc.make_triples(E, R, n) if case == "bench-shape" else _edge_triples(E, n, seed=3)
    ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
    s, p, o = ct[:, 0].contiguous(), ct[:, 1].contiguous(), ct[:, 2].contiguous()
    got = eng.train_1vsall_forward(model, ce, cr, ct, loss)
    sp_po = eng.score_sp_po(model, ce, cr, s, p, o)
    z = torch.cat([sp_po[:, :E], sp_po[:, E:]], 0)
    _step_check(eng, sms, f"{model} E={E} D={D} n={n} {case} {loss}", loss, got, z, torch.cat([o, s]), n)
    ref = orc.train_1vsall_forward(model, ce.double(), cr.double(), ct, loss)
    _rel_close(got, ref, f"{case} {loss} vs fp64 scores")


@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_fused_reciprocal_step_total(eng, sms, loss):
    """The reciprocal-relations step: rows n..2n are the sp_ queries (o, p + R), labelled s."""
    model, E, D, n = "distmult", 3001, 256, 389
    ent, rel2 = orc.make_tables(model, E, 2 * R, D, sigma=0.5)
    tri = _edge_triples(E, n, seed=4)
    ce, cr, ct = ent.cuda(), rel2.cuda(), tri.cuda()
    s, p, o = ct[:, 0].contiguous(), ct[:, 1].contiguous(), ct[:, 2].contiguous()
    got = eng.train_1vsall_reciprocal_forward(model, ce, cr, ct, R, loss)
    z = eng.score_1vsN(model, "sp_", ce, cr, ce, torch.cat([s, o]), torch.cat([p, p + R]))
    _step_check(eng, sms, f"reciprocal {model} {loss}", loss, got, z, torch.cat([o, s]), n)
    zref = orc.reciprocal_score_sp_po(model, ce.double(), cr.double(), s, p, o, R)
    fn = (lambda x, y: orc.bce_loss(x, y)) if loss == "bce" else orc.kl_loss
    ref = (fn(zref[:, :E], o) + fn(zref[:, E:], s)) / n
    _rel_close(got, ref, f"reciprocal {loss} vs fp64 scores")
