"""The tensor-core scorer's schedule and register epilogue (pairwise_tc.cu) against the fp64 oracle.

The shapes are chosen for the persistent schedule: CTA ranges that straddle query tiles, ranges of odd and even
length (so the two ping-pong consumer warpgroups get equal or unequal shares, or one gets none), fewer tiles than
SMs, reduction lengths of 1, 4, 8 and 16 K chunks around the 3-stage ring, and n = 4096.  Bars: scores 1e-4 * rms,
losses 1e-4 relative, rank / tie counts bit-exact on the kernel's own scores."""
import pytest
import torch

from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4

# (model, E, D, n): D sets the padded reduction (ComplEx / DistMult K = D): 64, 256, 512, 1024
SHAPES = [
    ("complex", 100, 32, 16),        # one tile: a single CTA, the second consumer warpgroup idle
    ("complex", 1000, 256, 100),     # 16 tiles < SMs: one tile per CTA
    ("distmult", 6007, 512, 389),    # 7 x 47 tiles: ranges of 2 and 3 tiles straddling query tiles
    ("complex", 3001, 1024, 77),     # 16 K chunks per tile, ring wraps within a tile
    ("complex", 1000, 64, 4096),     # n = 4096
]
IDS = [f"{m}-E{e}-D{d}-n{n}" for m, e, d, n in SHAPES]


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    return engine


def _assert_close(got, ref, what, tol=TOL):
    got, ref = got.detach().cpu().double(), ref.double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    err = float((got - ref).abs().max())
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e}"


def _rel_close(got, ref, what, tol=TOL):
    got, ref = float(got), float(ref)
    assert abs(got - ref) <= tol * abs(ref), f"{what}: {got} vs {ref}"


def _problem(model, E, D, n, sigma=1.0):
    ent, rel = orc.make_tables(model, E, 11, D, sigma=sigma)
    tri = orc.make_triples(E, 11, n)
    return ent, rel, tri, ent.cuda(), rel.cuda(), tri.cuda()


def _spo(t):
    return t[:, 0].contiguous(), t[:, 1].contiguous(), t[:, 2].contiguous()


def _multi_hot(n, m, seed):
    g = torch.Generator().manual_seed(seed)
    dense = (torch.rand((n, m), generator=g) < 0.01).float()
    dense[torch.arange(n), torch.randint(0, m, (n,), generator=g)] = 1.0   # every row has a positive
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = dense.sum(1).long().cumsum(0)
    cols = dense.nonzero()[:, 1].contiguous()
    return dense, offs, cols


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_store_sp_po(eng, shape):
    """Plain store epilogue, both directions stacked (the sp|po seam sits inside a query tile when n % 64 != 0)."""
    model, E, D, n = shape
    ent, rel, tri, ce, cr, ct = _problem(model, E, D, n)
    s, p, o = _spo(ct)
    ref = orc.score_sp_po(model, ent.double(), rel.double(), tri[:, 0], tri[:, 1], tri[:, 2])
    _assert_close(eng.score_sp_po(model, ce, cr, s, p, o), ref, "sp_po")


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_loss_index_labels(eng, shape, loss):
    model, E, D, n = shape
    ent, rel, tri, ce, cr, ct = _problem(model, E, D, n)
    ref = orc.train_1vsall_forward(model, ent.double(), rel.double(), tri, loss)
    _rel_close(eng.train_1vsall_forward(model, ce, cr, ct, loss), ref, f"{loss} index labels")


@pytest.mark.parametrize("n,E,D", [(32, 25000, 128), (48, 28000, 128), (64, 30000, 256)])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_loss_one_query_tile_many_entity_tiles(eng, n, E, D, loss):
    """One query tile against 196-235 entity tiles: more tiles than SMs, one tile per CTA.  The per-row partial slots
    must stay within the workspace the library sizes (at most two per CTA)."""
    ent, rel, tri, ce, cr, ct = _problem("complex", E, D, n)
    ref = orc.train_1vsall_forward("complex", ent.double(), rel.double(), tri, loss)
    _rel_close(eng.train_1vsall_forward("complex", ce, cr, ct, loss), ref, f"{loss} n={n} E={E}")


@pytest.mark.parametrize("n", [389, 1100])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_loss_dense_and_csr_labels(eng, n, loss):
    model, E, D = "complex", 3001, 256
    ent, rel, tri, ce, cr, ct = _problem(model, E, D, n, sigma=0.3)
    s, p, _ = _spo(ct)
    dense, offs, cols = _multi_hot(n, E, seed=n)
    scores = orc.score_sp(model, ent.double(), rel.double(), tri[:, 0], tri[:, 1])
    ref = orc.bce_loss(scores, dense.double()) if loss == "bce" else orc.kl_loss(scores, dense.double())
    got_dense = eng.score_1vsN_loss(model, "sp_", ce, cr, ce, dense.cuda(), s, p, None, loss)
    _rel_close(got_dense, ref, f"{loss} dense labels")
    got_csr = eng.score_1vsN_loss_csr(model, "sp_", ce, cr, ce, offs.cuda(), cols.cuda(), s, p, loss)
    _rel_close(got_csr, ref, f"{loss} CSR labels")


@pytest.mark.parametrize("shape", SHAPES[1:4], ids=IDS[1:4])
def test_rank_dense_and_csr_filters(eng, shape):
    model, E, D, n = shape
    _, _, _, ce, cr, ct = _problem(model, E, D, n)
    s, p, o = _spo(ct)
    sp_po = eng.score_sp_po(model, ce, cr, s, p, o).cpu()
    scores = torch.cat([sp_po[:, :E], sp_po[:, E:]], 0)                        # stacked [2n, E]
    own = torch.cat([o.cpu(), s.cpu()])
    true = scores[torch.arange(2 * n), own].clone()
    dense, offs, cols = _multi_hot(2 * n, E, seed=7)
    dense[torch.arange(2 * n), own] = 0.0                                        # the dense filter leaves the answer in
    filt = dense * float("inf")
    filt[dense == 0] = 0.0
    rr, tt = orc.ranks_and_ties(scores - filt, true)
    r, t = eng.rank_sp_po(model, ce, cr, ce, ce, true.cuda(), s, p, o, filter_labels=filt.cuda())
    assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)
    # CSR filter: the same columns plus the answer, which own_col keeps in
    dense[torch.arange(2 * n), own] = 1.0
    offs = torch.zeros(2 * n + 1, dtype=torch.int64)
    offs[1:] = dense.sum(1).long().cumsum(0)
    cols = dense.nonzero()[:, 1].contiguous()
    r, t = eng.rank_sp_po_csr(model, ce, cr, ce, ce, true.cuda(), offs.cuda(), cols.cuda(), own.cuda(), s, p, o)
    assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)


@pytest.mark.parametrize("M,N,K", [(300, 700, 1200), (2048, 1000, 200)])
def test_gemm_nt(eng, M, N, K):
    """gemm_nt: K > 512 runs the split-K work items (fp32 red.add of 512-wide segments)."""
    g = torch.Generator().manual_seed(M)
    a, b = torch.randn((M, K), generator=g), torch.randn((N, K), generator=g)
    _assert_close(eng.gemm_nt(a.cuda(), b.cuda()), a.double() @ b.double().T, "gemm_nt")


def test_repeatable(eng):
    """Fixed-order reductions: the same call twice gives the same bits."""
    model, E, D, n = SHAPES[2]
    _, _, _, ce, cr, ct = _problem(model, E, D, n)
    s, p, o = _spo(ct)
    for loss in ("bce", "kl"):
        a = eng.train_1vsall_forward(model, ce, cr, ct, loss).item()
        b = eng.train_1vsall_forward(model, ce, cr, ct, loss).item()
        assert a == b, (loss, a, b)
    assert torch.equal(eng.score_sp_po(model, ce, cr, s, p, o), eng.score_sp_po(model, ce, cr, s, p, o))
