"""Embedding dropout on the H100 at the shapes where its kernels change code path: the mask kernel at table scale and at
element indexes up to the 2^48 limit, and the 1vsAll, KvsAll and negative-sampling dropout entry points against fp64
autograd of the masked reference expression at multi-tile, split-K and full-size shapes.  tests/test_gpu_dropout.py and
tests/test_gpu_ns_dropout.py check the same entry points at toy shapes; the references here draw their masks with the
vectorised mirror of tests/philox_np.py, which tests/test_dropout_mirror_cpu.py pins to the scalar one bit for bit."""
import pytest
import torch

import dropout_oracle as dro
import ns_dropout_oracle as nso
import philox_np
from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4          # of the reference's rms, as tests/test_gpu_dropout.py
LIM = 2 ** 48       # element indexes row * dim + k of a draw stay below this (validate_dropout, capi.cu)
# d_ent where a few rows sum thousands of fp32 terms while most rows sum few, so max/rms is large:
# - Dot family at E >= 5003: the query rows' gradient dQ = G T reduces over all E candidates.  Its error relative to
#   the largest query-row gradient is the same with and without dropout (2.5e-6 for ComplEx d=256, E=5003, n=600).
#   Dropout at p_ent = 0.4 raises max/rms from 28 to 41 there, so the same relative error is a larger share of the
#   rms.  Measured on an H100 against fp64 on the same tables: the dropout-free fused step gives 0.70e-4 of rms at
#   E=5003 and 0.96e-4 at E=14541; the dropout route gives the same at rates 0, and up to 1.7e-4 (E=5003) and 2.1e-4
#   (E=14541) at rates 0.4 / 0.2.
# - Negative sampling at K = 1000: each fixed row of a slot's block receives K contributions, added with atomics in a
#   run-dependent order; CP's `triple` O slot passed TOL in one run and gave 1.09e-4 in the next.
# A wrong row, column, mask or split-K segment moves whole gradient elements, which is of order 1 in this ratio.
# test_1vsall_dropout_rate_zero_is_the_fused_step holds the 1vsAll route to TOL against the fused step itself.
TOL_LONG = 3e-4


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


@pytest.fixture(autouse=True)
def fast_mirror(monkeypatch):
    """The references draw their masks with the vectorised mirror; ns_dropout_oracle calls dro.mask through the module,
    so it follows."""
    monkeypatch.setattr(dro, "mask", philox_np.mask)


def _close(got, ref, what, tol=TOL):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = float((got - ref).abs().max())
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


# ---- a. the mask kernel ------------------------------------------------------------------------------------------
def test_mask_kernel_at_table_scale(eng):
    """One table draw at the bench shape (14 541 x 512): 1.86 M Philox blocks, 7 270 CTAs."""
    args = (0.4, 2 ** 63 + 2024, 2 ** 32 + 77, 2, 14541, 512, 0)
    assert torch.equal(eng.dropout_mask(*args).cpu().bool(), philox_np.mask(*args))


@pytest.mark.parametrize("dim,stream,seed,call", [(66, 3, 2 ** 63 + 11, 2 ** 32 + 1), (512, 17, 2 ** 64 - 1, 2 ** 40 + 7)])
def test_mask_kernel_across_2_34(eng, dim, stream, seed, call):
    """Rows whose element indexes cross 2^34: group index e >> 2 crosses 2^32, so the counter's high word carries group
    bits next to the stream bits; dim 66 makes blocks straddle rows.  Stream 17 is one of the negative-sampling draws."""
    rows = 4099
    row_base = 2 ** 34 // dim - rows // 2
    assert row_base * dim < 2 ** 34 < (row_base + rows) * dim
    args = (0.3, seed, call, stream, rows, dim, row_base)
    assert torch.equal(eng.dropout_mask(*args).cpu().bool(), philox_np.mask(*args))


@pytest.mark.parametrize("dim", [66, 512])
def test_mask_kernel_at_the_2_48_limit(eng, dim):
    """The last rows a draw may address are accepted and drawn as the mirror draws them; one row further is refused."""
    rows = 7
    row_base = LIM // dim - rows                               # (row_base + rows) * dim <= 2^48, exactly for dim 512
    args = (0.5, 2 ** 63 + 3, 2 ** 33 + 5, 4, rows, dim, row_base)
    assert torch.equal(eng.dropout_mask(*args).cpu().bool(), philox_np.mask(*args))
    with pytest.raises(ValueError):
        eng.dropout_mask(0.5, 2 ** 63 + 3, 2 ** 33 + 5, 4, rows, dim, row_base + 1)


# ---- b. 1vsAll ---------------------------------------------------------------------------------------------------
class _ModulusL1(torch.autograd.Function):
    """-sum_k |q_k - t_k| over complex elements with the kernels' convention at |q_k - t_k| = 0: gradient 0, where the
    reference expression's sqrt gives NaN (dropout makes such ties common)."""

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


def _problem_1vsall(model, E, D, n, sigma, R=11):
    ent, rel = orc.make_tables(model, E, R, D, sigma=sigma)
    tri = orc.make_triples(E, R, n, seed=7)
    tri[5] = tri[4]                                            # a duplicated triple
    tri[9, 2] = tri[9, 0]                                      # s == o
    return ent, rel, tri


def _key(eng):
    return eng.DropoutKey(0.4, 0.2, seed=2 ** 63 + 2024, call=2 ** 32 + 77, row_base=1000)


def _check_1vsall(eng, model, l_norm, loss, ent, rel, tri, key, ent_tol=TOL):
    offset = 0.5 if loss == "bce" else 0.0
    val, de, dr = dro.grads(lambda e, r: _ref_1vsall(model, e, r, tri, loss, offset, key, l_norm),
                            ent.double(), rel.double())
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    got = eng.train_1vsall_forward(model, ec, rc, tc, loss, offset, l_norm, dropout=key)
    assert float(got) == pytest.approx(float(val), rel=TOL)
    ge, gr = eng.train_1vsall_backward(model, ec, rc, tc, loss, offset, l_norm, dropout=key)
    _close(ge, de, f"{model} {loss} d_ent", tol=ent_tol)
    _close(gr, dr, f"{model} {loss} d_rel")


# Dot family at E = 5003, n = 600: round_up(n, 64) = 640 and round_up(E, 64) = 5056 both exceed 512, so the dT (over n)
# and dQ (over E) GEMMs both run split-K (gemm_planes); E and n are ragged against the 64-row tiles, and the folded
# widths K (ComplEx / SimplE / DistMult: D, CP: D / 2 = 128, RESCAL: D = 48) span several 64-wide chunks (RESCAL: a
# ragged one).  CP's K = 128 >= 32 puts it on the tensor cores, and its dT lands in the column half [col_off, col_off
# + K) of dropout_add_cols.
DOT = [("complex", 256), ("distmult", 192), ("simple", 256), ("cp", 256), ("rescal", 48)]
E1, N1 = 5003, 600


@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,D", DOT)
def test_1vsall_dropout_dot_family_split_k(eng, model, D, loss):
    assert -(-N1 // 64) * 64 > 512 and -(-E1 // 64) * 64 > 512
    ent, rel, tri = _problem_1vsall(model, E1, D, N1, 0.3)
    _check_1vsall(eng, model, 1.0, loss, ent, rel, tri, _key(eng), ent_tol=TOL_LONG)


# Distance family at E = 1201, n = 139, D = 136: the row-gradient passes walk 64-float chunks of K (TransE 136, RotatE
# 68 complex elements), the last one ragged; E and n are ragged against the scorer's tiles.
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,l_norm", [("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)])
def test_1vsall_dropout_distance_family(eng, model, l_norm, loss):
    ent, rel, tri = _problem_1vsall(model, 1201, 136, 139, 0.3)
    _check_1vsall(eng, model, l_norm, loss, ent, rel, tri, _key(eng))


# The bench and README shape: ComplEx d = 512, E = 14 541, batch 1024.
EF, DF, NF = 14541, 512, 1024


@pytest.fixture(scope="module")
def fullsize():
    return _problem_1vsall("complex", EF, DF, NF, 0.2)


@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_1vsall_dropout_full_size(eng, fullsize, loss):
    _check_1vsall(eng, "complex", 1.0, loss, *fullsize, _key(eng), ent_tol=TOL_LONG)


@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_1vsall_dropout_rate_zero_is_the_fused_step(eng, fullsize, loss):
    """Rates 0 run the dropout route (gathers, scratch dT, scatters) on unmasked operands: the loss and gradients are
    those of the dropout-free fused step."""
    ent, rel, tri = fullsize
    ec, rc, tc = ent.cuda(), rel.cuda(), tri.cuda()
    offset = 0.5 if loss == "bce" else 0.0
    key = eng.DropoutKey(0.0, 0.0, seed=5, call=2 ** 32 + 1, row_base=1000)
    want = float(eng.train_1vsall_forward("complex", ec, rc, tc, loss, offset))
    got = float(eng.train_1vsall_forward("complex", ec, rc, tc, loss, offset, dropout=key))
    assert got == pytest.approx(want, rel=TOL)
    we, wr = eng.train_1vsall_backward("complex", ec, rc, tc, loss, offset)
    ge, gr = eng.train_1vsall_backward("complex", ec, rc, tc, loss, offset, dropout=key)
    _close(ge, we, "d_ent")
    _close(gr, wr, "d_rel")


# ---- c. KvsAll ---------------------------------------------------------------------------------------------------
def _csr(n, E, seed=11):
    """CSR labels with an empty row, a duplicate column (label 2), the columns 0, 127, 128 and E - 1 (tile and table
    edges) and one row of 900 columns; 1-5 random columns elsewhere."""
    g = torch.Generator().manual_seed(seed)
    rows = [torch.sort(torch.randint(0, E, (int(c),), generator=g))[0]
            for c in torch.randint(1, 6, (n,), generator=g)]
    rows[3] = torch.zeros(0, dtype=torch.int64)
    rows[5] = torch.tensor([17, 40, 40, 41])
    rows[8] = torch.tensor([0, 127, 128, E - 1])
    rows[n - 2] = torch.sort(torch.randperm(E, generator=g)[:900])[0]
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.tensor([len(r) for r in rows]), 0)
    return offs, torch.cat(rows)


@pytest.mark.parametrize("eps", [0.0, 0.2])
@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("combine", ["sp_", "_po"])
@pytest.mark.parametrize("model,D", DOT)
def test_kvsall_dropout_split_k(eng, model, D, combine, loss, eps):
    ent, rel, tri = _problem_1vsall(model, E1, D, N1, 0.3)
    q, p = tri[:, 0], tri[:, 1]
    offs, cols = _csr(N1, E1)
    key = _key(eng)
    offset = 0.5 if loss == "bce" else 0.0
    bs = 2 * N1
    val, de, dr = dro.grads(lambda e, r: dro.loss_kvsall(model, combine, e, r, q, p, offs, cols, loss, offset, eps, key)
                            / bs, ent.double(), rel.double())
    ec, rc = ent.cuda(), rel.cuda()
    qc, pc, oc, cc = q.cuda(), p.cuda(), offs.cuda(), cols.cuda()
    got = eng.score_1vsN_loss_csr(model, combine, ec, rc, ec, oc, cc, qc, pc, loss, offset, eps, dropout=key) / bs
    assert float(got) == pytest.approx(float(val), rel=TOL)
    ge, gr = eng.score_1vsN_loss_csr_backward(model, combine, ec, rc, qc, pc, oc, cc, loss, offset, eps, bs, dropout=key)
    _close(ge, de, f"{model} {combine} d_ent", tol=TOL_LONG)
    _close(gr, dr, f"{model} {combine} d_rel")


# ---- d. negative sampling ----------------------------------------------------------------------------------------
NS_CASES = [("complex", 1.0), ("distmult", 1.0), ("simple", 1.0), ("cp", 1.0), ("rescal", 1.0), ("transe", 1.0),
            ("transe", 2.0), ("rotate", 1.0)]
EN = 5003


def _ns_problem(model, D, N, K, seed=0):
    ent, rel = orc.make_tables(model, EN, 7, D, sigma=0.3, seed=seed)
    tri = orc.make_triples(EN, 7, N, seed=seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    neg = torch.randint(0, EN, (N, K), generator=g)          # N K > E: ids repeat within and across rows
    neg[:, 3] = neg[:, 4]
    neg[1, :50] = neg[0, :50]
    return ent, rel, tri, neg


def _ns_key(eng):
    return eng.DropoutKey(0.3, 0.2, seed=2 ** 63 + 1234567, call=2 ** 32 + 9, row_base=4093)


def _grad_with_zeros(N, K, seed=3):
    g = torch.Generator().manual_seed(seed)
    G = torch.randn(N, K + 1, generator=g)
    G[G.abs() < 0.3] = 0.0                                     # the kernels skip g == 0
    return G


def _check_ns(eng, model, l_norm, slot, impl, ent, rel, tri, neg, key, G=None, ent_tol=TOL):
    """Scores against the fp64 block, then the backward of G (random unless given) against autograd of <G, block>."""
    e32, r32 = ent.cuda(), rel.cuda()
    scores = eng.ns_score(model, e32, r32, tri.cuda(), neg.cuda(), slot, True, l_norm, dropout=key,
                          implementation=impl)
    e, r = ent.double().requires_grad_(True), rel.double().requires_grad_(True)
    with torch.enable_grad():
        ref = nso.block(model, e, r, tri, slot, neg, key, impl, l_norm)
        _close(scores, ref.detach(), f"{model} slot {slot} {impl} scores")
        if G is None:
            G = _grad_with_zeros(*neg.shape)
        de, dr = torch.autograd.grad((G.double().cpu() * ref).sum(), (e, r))
    d_ent, d_rel = eng.ns_backward(model, e32, r32, tri.cuda(), {slot: neg.cuda()}, l_norm=l_norm,
                                   grad_scores={slot: G.cuda()}, dropout=key, implementation=impl)
    _close(d_ent, de, f"{model} slot {slot} {impl} d_ent", tol=ent_tol)
    _close(d_rel, dr, f"{model} slot {slot} {impl} d_rel")
    return scores


# K = 1000 > NS_PER_BLOCK = 256 (rowwise.cu): four forward CTAs per row; K > NSB_PER_BLOCK = 64 (grad.cu): 16 backward
# blocks per row combine the masked dq.  D = 256 is 64 float4 columns per row: every lane of a warp loops, and the
# masked column col_off + 4k runs past the first pass.  RESCAL reads its D^2 relation row per triple: D = 32, N = 9,
# K = 300 (still two forward CTAs and five backward blocks per row).
@pytest.mark.parametrize("impl", ["triple", "batch"])
@pytest.mark.parametrize("slot", [0, 2])
@pytest.mark.parametrize("model,l_norm", NS_CASES)
def test_ns_dropout_production_shape(eng, model, l_norm, slot, impl):
    D, N, K = (32, 9, 300) if model == "rescal" else (256, 37, 1000)
    ent, rel, tri, neg = _ns_problem(model, D, N, K)
    neg[:, 0] = tri[:, slot]                                   # a negative equal to the positive
    _check_ns(eng, model, l_norm, slot, impl, ent, rel, tri, neg, _ns_key(eng), ent_tol=TOL_LONG)


@pytest.mark.parametrize("slot", [0, 2])
def test_ns_dropout_complex_batch_at_d_1024(eng, slot):
    """D = 1024 is the widest `batch` serves: every lane holds all NSB_MAXK / 32 = 32 dq registers."""
    ent, rel, tri, neg = _ns_problem("complex", 1024, 9, 300, seed=4)
    _check_ns(eng, "complex", 1.0, slot, "batch", ent, rel, tri, neg, _ns_key(eng), ent_tol=TOL_LONG)


@pytest.mark.parametrize("impl", ["triple", "batch"])
def test_ns_dropout_kl_end_to_end(eng, impl):
    """G from ns_loss (kl) of the kernel's own scores, as the training step takes it."""
    ent, rel, tri, neg = _ns_problem("complex", 256, 37, 1000, seed=6)
    key = _ns_key(eng)
    scores = eng.ns_score("complex", ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda(), 2, True, dropout=key,
                          implementation=impl)
    _, G = eng.ns_loss(scores, "kl", batch_size=37, want_grad=True)
    _check_ns(eng, "complex", 1.0, 2, impl, ent, rel, tri, neg, key, G=G.cpu(), ent_tol=TOL_LONG)
