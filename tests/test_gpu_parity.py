"""GPU parity tests: the CUDA path (through the C ABI) vs the CPU oracle and vs golden vectors
generated from the live reference.  Tolerance for floating point: max|d| <= 1e-4 * rms(reference)
(north_star: "within 1e-4 relative fp32"); integer outputs (ranks/ties) bit-exact."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
S, P, O = 0, 1, 2
TOL = 1e-4


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    assert engine.device_ok(), "libb200kge needs an sm_90 (H100) device"
    return engine


def _load(name):
    z = np.load(os.path.join(GOLDEN, name))
    return {k: torch.from_numpy(z[k]) if z[k].ndim else z[k].item() for k in z.files}


def _assert_close(got, ref, what, tol=TOL):
    got = got.detach().cpu().double()
    ref = ref.double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    err = float((got - ref).abs().max()) if ref.numel() else 0.0
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e} ratio={err / rms:.2e}"


SCORE_FILES = sorted(os.path.basename(f) for f in glob.glob(os.path.join(GOLDEN, "scores_*.npz")))


@pytest.mark.parametrize("fname", SCORE_FILES)
def test_golden_scores(eng, fname):
    g = _load(fname)
    model = fname[len("scores_"):-4].split("_")[0]
    ln = float(g["l_norm"])
    ent, rel, tri = g["ent"].cuda(), g["rel"].cuda(), g["triples"].cuda()
    s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
    sub = g["subset"].cuda()
    _assert_close(eng.score_spo(model, ent, rel, ent, s, p, o, ln), g["spo"], "spo")
    _assert_close(eng.score_1vsN(model, "sp_", ent, rel, ent, s, p, None, ln), g["sp"], "sp")
    _assert_close(eng.score_1vsN(model, "_po", ent, rel, ent, o, p, None, ln), g["po"], "po")
    _assert_close(eng.score_1vsN(model, "sp_", ent, rel, ent, s, p, sub, ln), g["sp_subset"], "sp_subset")
    _assert_close(eng.score_1vsN(model, "_po", ent, rel, ent, o, p, sub, ln), g["po_subset"], "po_subset")
    _assert_close(eng.score_sp_po(model, ent, rel, s, p, o, None, ln), g["sp_po"], "sp_po")
    _assert_close(eng.score_sp_po(model, ent, rel, s, p, o, sub, ln), g["sp_po_subset"], "sp_po_subset")
    # RelationalScorer.score_emb form: already-gathered embeddings, no indexes
    _assert_close(eng.score_1vsN(model, "sp_", ent[s], rel[p], ent[sub], l_norm=ln), g["sp_subset"], "score_emb sp_")
    _assert_close(eng.score_spo(model, ent[s], rel[p], ent[o], l_norm=ln), g["spo"], "score_emb spo")


def test_golden_scores_tensor_core(eng):
    """Forces the 3xTF32 tensor-core kernel on the golden cases it can take (dot family, K >= 32)."""
    for fname, model in (("scores_complex.npz", "complex"), ("scores_distmult.npz", "distmult"),
                         ("scores_simple.npz", "simple"), ("scores_complex_sigma01.npz", "complex")):
        g = _load(fname)
        ent, rel, tri = g["ent"].cuda(), g["rel"].cuda(), g["triples"].cuda()
        s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
        sub = g["subset"].cuda()
        _assert_close(eng.score_1vsN(model, "sp_", ent, rel, ent, s, p, None, precision="3xtf32"), g["sp"], fname + " sp tc")
        _assert_close(eng.score_1vsN(model, "_po", ent, rel, ent, o, p, sub, precision="3xtf32"), g["po_subset"], fname + " po_subset tc")
        _assert_close(eng.score_sp_po(model, ent, rel, s, p, o, None, precision="3xtf32"), g["sp_po"], fname + " sp_po tc")
        _assert_close(eng.score_sp_po(model, ent, rel, s, p, o, None, precision="tf32+bf16x2"), g["sp_po"], fname + " sp_po mixed")


MEDIUM = [("complex", 128), ("distmult", 128), ("simple", 128), ("cp", 128), ("rescal", 48),
          ("transe", 128), ("rotate", 128)]


@pytest.mark.parametrize("model,D", MEDIUM)
@pytest.mark.parametrize("sigma", [1.0, 0.1])
def test_oracle_medium(eng, model, D, sigma):
    E, R, n = 5003, 11, 301          # odd sizes: ragged tiles everywhere
    ent, rel = orc.make_tables(model, E, R, D, sigma=sigma)
    tri = orc.make_triples(E, R, n)
    ref = orc.score_sp_po(model, ent, rel, tri[:, S], tri[:, P], tri[:, O])
    ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
    s, p, o = ct[:, S].contiguous(), ct[:, P].contiguous(), ct[:, O].contiguous()
    precs = ["auto", "fp32"] + (["3xtf32", "tf32+bf16x2"] if model in ("complex", "distmult", "simple", "rescal") else [])
    for prec in precs:
        got = eng.score_sp_po(model, ce, cr, s, p, o, precision=prec)
        _assert_close(got, ref, f"{model} sp_po {prec}")
    ref_spo = orc.score_spo(model, ent, rel, tri[:, S], tri[:, P], tri[:, O])
    _assert_close(eng.score_spo(model, ce, cr, ce, s, p, o), ref_spo, f"{model} spo")


def test_tensor_core_kernel_variants(eng):
    """In-kernel split of raw fp32 operands in the 3xTF32 and the mixed split modes: dense scores, fused BCE/KL,
    fused rank counting; ragged sizes (tiles cut in both dimensions, odd number of query tiles)."""
    for model, D, prec in (("complex", 192, "3xtf32"), ("complex", 192, "tf32+bf16x2"), ("distmult", 64, "tf32+bf16x2"),
                           ("rescal", 40, "3xtf32"), ("rescal", 40, "tf32+bf16x2")):
        E, R, n = 6007, 7, 389
        ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
        tri = orc.make_triples(E, R, n)
        ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
        s, p, o = ct[:, S].contiguous(), ct[:, P].contiguous(), ct[:, O].contiguous()
        ref = orc.score_sp_po(model, ent, rel, tri[:, S], tri[:, P], tri[:, O])
        got = eng.score_sp_po(model, ce, cr, s, p, o, precision=prec)
        _assert_close(got, ref, f"{model} sp_po {prec}")
        sub = torch.randperm(E, generator=torch.Generator().manual_seed(1))[:1500]
        got = eng.score_1vsN(model, "_po", ce, cr, ce, o, p, sub.cuda(), precision=prec)
        _assert_close(got, orc.score_po(model, ent, rel, tri[:, P], tri[:, O], sub), f"{model} po subset {prec}")
        for loss, fn in (("bce", orc.bce_loss), ("kl", orc.kl_loss)):
            refl = float(orc.train_1vsall_forward(model, ent, rel, tri, loss))
            gotl = float(eng.train_1vsall_forward(model, ce, cr, ct, loss, precision=prec))
            assert abs(gotl - refl) <= 1e-4 * abs(refl), (model, loss, prec, gotl, refl)
        dense = eng.score_1vsN(model, "sp_", ce, cr, ce, s, p, precision=prec)
        true = dense[torch.arange(n, device="cuda"), o].clone()
        rr, tt = orc.ranks_and_ties(dense.cpu(), true.cpu())
        r, t = eng.score_1vsN_rank(model, "sp_", ce, cr, ce, true, s, p, precision=prec)
        assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)


def test_tf32_single_pass_is_loose_but_sane(eng):
    ent, rel = orc.make_tables("complex", 4099, 7, 256)
    tri = orc.make_triples(4099, 7, 256)
    ref = orc.score_sp(  "complex", ent, rel, tri[:, S], tri[:, P])
    got = eng.score_1vsN("complex", "sp_", ent.cuda(), rel.cuda(), ent.cuda(), tri[:, S].cuda(), tri[:, P].cuda(),
                         precision="tf32")
    _assert_close(got, ref, "tf32 1-pass", tol=1e-2)


@pytest.mark.parametrize("model,D", [("complex", 128), ("rescal", 32), ("transe", 64), ("rotate", 64)])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_fused_loss_vs_oracle(eng, model, D, loss):
    E, R, n = 3001, 5, 200
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.3)
    tri = orc.make_triples(E, R, n)
    s, p, o = tri[:, S], tri[:, P], tri[:, O]
    sc_sp = orc.score_sp(model, ent, rel, s, p)
    sc_po = orc.score_po(model, ent, rel, p, o)
    g = torch.Generator().manual_seed(3)
    multi = (torch.rand((n, E), generator=g) < 0.01).float()
    multi[torch.arange(n), o] = 1.0
    smooth = orc.kvsall_smooth_labels(multi, 0.1)
    ce, cr = ent.cuda(), rel.cuda()
    off = 1.5 if loss == "bce" else 0.0
    fn = (lambda x, y: orc.bce_loss(x, y, off)) if loss == "bce" else orc.kl_loss
    precs = ["auto", "fp32"]
    for prec in precs:
        # index labels (1vsAll)
        got = eng.score_1vsN_loss(model, "sp_", ce, cr, ce, o.cuda(), s.cuda(), p.cuda(), None, loss, off, precision=prec)
        ref = fn(sc_sp, o)
        assert abs(float(got) - float(ref)) <= 1e-4 * abs(float(ref)), (model, loss, prec, float(got), float(ref))
        got = eng.score_1vsN_loss(model, "_po", ce, cr, ce, s.cuda(), o.cuda(), p.cuda(), None, loss, off, precision=prec)
        ref = fn(sc_po, s)
        assert abs(float(got) - float(ref)) <= 1e-4 * abs(float(ref)), (model, loss, prec, float(got), float(ref))
        # dense labels (KvsAll multi-hot, with label smoothing)
        for lab in (multi, smooth):
            got, rows = eng.score_1vsN_loss(model, "sp_", ce, cr, ce, lab.cuda(), s.cuda(), p.cuda(), None, loss, off,
                                            precision=prec, return_rows=True)
            ref = fn(sc_sp, lab)
            assert abs(float(got) - float(ref)) <= 1e-4 * abs(float(ref)), (model, loss, prec, float(got), float(ref))
            assert abs(float(rows.sum()) - float(ref)) <= 1e-4 * abs(float(ref))


def test_dense_loss_vs_golden_and_oracle(eng):
    g = _load("losses.npz")
    x = g["scores"].cuda()
    rel = lambda a, b: abs(float(a) - float(b)) <= 1e-5 * max(1.0, abs(float(b)))
    assert rel(eng.loss_dense(x, g["idx"].cuda(), "bce"), g["bce_idx"])
    assert rel(eng.loss_dense(x, g["idx"].cuda(), "bce", 2.0), g["bce_idx_off2"])
    assert rel(eng.loss_dense(x, g["multi"].cuda(), "bce"), g["bce_multi"])
    assert rel(eng.loss_dense(x, g["smooth"].cuda(), "bce"), g["bce_smooth"])
    assert rel(eng.loss_dense(x, g["idx"].cuda(), "kl"), g["kl_idx"])
    assert rel(eng.loss_dense(x, g["multi"].cuda(), "kl"), g["kl_multi"])
    assert rel(eng.loss_dense(x, g["smooth"].cuda(), "kl"), g["kl_smooth"])
    # larger, ragged
    gen = torch.Generator().manual_seed(1)
    x = torch.randn((77, 9001), generator=gen) * 4
    idx = torch.randint(0, 9001, (77,), generator=gen)
    for loss, fn in (("bce", orc.bce_loss), ("kl", orc.kl_loss)):
        got, rows = eng.loss_dense(x.cuda(), idx.cuda(), loss, return_rows=True)
        ref = fn(x, idx)
        assert abs(float(got) - float(ref)) <= 1e-5 * abs(float(ref))
        assert rows.shape == (77,)


def test_rank_dense_bit_exact(eng):
    g = _load("ranks.npz")
    r, t = eng.rank_dense(g["sp"].cuda(), g["o_true"].cuda())
    assert torch.equal(r.cpu(), g["raw_o_rank"]) and torch.equal(t.cpu(), g["raw_o_ties"])
    r, t = eng.rank_dense(g["po"].cuda(), g["s_true"].cuda())
    assert torch.equal(r.cpu(), g["raw_s_rank"]) and torch.equal(t.cpu(), g["raw_s_ties"])
    E = g["sp"].shape[1]
    lab = g["labels"].cuda()
    r, t = eng.rank_dense(g["sp"].cuda(), g["o_true"].cuda(), lab[:, :E])
    assert torch.equal(r.cpu(), g["filt_o_rank"]) and torch.equal(t.cpu(), g["filt_o_ties"])
    r, t = eng.rank_dense(g["po"].cuda(), g["s_true"].cuda(), lab[:, E:])
    assert torch.equal(r.cpu(), g["filt_s_rank"]) and torch.equal(t.cpu(), g["filt_s_ties"])
    # random large case with heavy ties, NaN and infinities vs the oracle
    gen = torch.Generator().manual_seed(9)
    x = torch.randn((64, 20011), generator=gen).round(decimals=2)
    x[3, 100:200] = float("nan")
    x[4, 50] = float("inf")
    x[5, :] = float("-inf")
    true = x[torch.arange(64), torch.randint(0, 20011, (64,), generator=gen)].clone()
    filt = torch.zeros_like(x)
    filt[torch.rand(x.shape, generator=gen) < 0.01] = float("inf")
    for f in (None, filt):
        rr, tt = orc.ranks_and_ties(x if f is None else x - f, true)
        r, t = eng.rank_dense(x.cuda(), true.cuda(), None if f is None else f.cuda())
        assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)
    # additivity over chunks (eval_entity_ranking.py:310-313)
    r = torch.zeros(64, dtype=torch.int64, device="cuda")
    t = torch.zeros(64, dtype=torch.int64, device="cuda")
    for c0 in range(0, 20011, 7000):
        eng.rank_dense(x[:, c0:c0 + 7000].cuda(), true.cuda(), rank=r, ties=t)
    rr, tt = orc.ranks_and_ties(x, true)
    assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)


@pytest.mark.parametrize("model,D,prec", [("complex", 128, "auto"), ("complex", 128, "fp32"), ("transe", 64, "auto"),
                                          ("rotate", 64, "auto"), ("rescal", 32, "auto")])
def test_fused_rank_equals_rank_of_own_scores(eng, model, D, prec):
    """Rank indices are bit-exact where that is well-posed: the fused score+rank kernel must return
    exactly the counts that the reference's rank arithmetic yields on the same kernel's scores."""
    E, R, n = 4001, 5, 150
    ent, rel = orc.make_tables(model, E, R, D)
    tri = orc.make_triples(E, R, n)
    ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
    s, p, o = ct[:, S].contiguous(), ct[:, P].contiguous(), ct[:, O].contiguous()
    for combine, q, tgt in (("sp_", s, o), ("_po", o, s)):
        dense = eng.score_1vsN(model, combine, ce, cr, ce, q, p, precision=prec)
        true = dense[torch.arange(n, device="cuda"), tgt].clone()
        gen = torch.Generator().manual_seed(2)
        filt = torch.zeros((n, E))
        filt[torch.rand((n, E), generator=gen) < 0.02] = float("inf")
        filt[torch.arange(n), tgt.cpu()] = 0.0
        for f in (None, filt):
            rr, tt = orc.ranks_and_ties(dense.cpu() if f is None else dense.cpu() - f, true.cpu())
            r, t = eng.score_1vsN_rank(model, combine, ce, cr, ce, true, q, p, None,
                                       None if f is None else f.cuda(), precision=prec)
            assert torch.equal(r.cpu(), rr), (model, combine, (r.cpu() - rr).abs().max())
            assert torch.equal(t.cpu(), tt)
    # end-to-end agreement with the oracle's own scores over more rows: two correct fp32 implementations with
    # different summation orders flip a few comparisons inside the isclose band (SURVEY 7.2: 0-2 of 512 rows even for a
    # plain fp32 reordering), never by more than one place; bench.py reports the measured rate at the headline shape
    n2 = 400
    tri2 = orc.make_triples(E, R, n2, seed=9)
    ct2 = tri2.cuda()
    ref = orc.score_sp(model, ent, rel, tri2[:, S], tri2[:, P])
    rr, tt = orc.ranks_and_ties(ref, ref[torch.arange(n2), tri2[:, O]])
    dense = eng.score_1vsN(model, "sp_", ce, cr, ce, ct2[:, S].contiguous(), ct2[:, P].contiguous(), precision=prec)
    r, t = eng.rank_dense(dense, dense[torch.arange(n2, device="cuda"), ct2[:, O]])
    final = orc.final_ranks(r.cpu(), t.cpu())
    agree = float((final == orc.final_ranks(rr, tt)).float().mean())
    assert agree >= 0.99, agree
    assert int((final - orc.final_ranks(rr, tt)).abs().max()) <= 1


@pytest.mark.parametrize("model", ["complex", "rotate", "transe", "rescal"])
def test_ns_golden(eng, model):
    g = _load(f"ns_{model}.npz")
    ln = float(g["l_norm"])
    ent, rel, tri = g["ent"].cuda(), g["rel"].cuda(), g["triples"].cuda()
    for slot, nm in ((S, "s"), (P, "p"), (O, "o")):
        got = eng.ns_score(model, ent, rel, tri, g[f"neg_{nm}"].cuda(), slot, False, ln)
        _assert_close(got, g[f"ns_{nm}_triple"], f"ns {model} {nm}")
        _assert_close(got, g[f"ns_{nm}_batch"], f"ns {model} {nm} (batch impl)")
        full = eng.ns_score(model, ent, rel, tri, g[f"neg_{nm}"].cuda(), slot, True, ln)
        _assert_close(full[:, 0], g["pos"], "ns positive column")
        _assert_close(full[:, 1:], g[f"ns_{nm}_triple"], "ns negatives columns")


@pytest.mark.parametrize("model,D", [("rotate", 128), ("complex", 128), ("transe", 128), ("distmult", 64)])
def test_ns_vs_oracle_medium(eng, model, D):
    E, R, n, K = 4093, 11, 64, 257
    ent, rel = orc.make_tables(model, E, R, D)
    tri = orc.make_triples(E, R, n)
    g = torch.Generator().manual_seed(4)
    for slot in (S, O):
        neg = torch.randint(0, E, (n, K), generator=g)
        ref = orc.ns_scores_with_positive(model, ent, rel, tri, neg, slot, "triple")
        got = eng.ns_score(model, ent.cuda(), rel.cuda(), tri.cuda(), neg.cuda(), slot, True)
        _assert_close(got, ref, f"ns {model} slot {slot}")


@pytest.mark.parametrize("model,D,loss", [("complex", 128, "bce"), ("complex", 128, "kl"), ("cp", 64, "bce"),
                                          ("transe", 64, "kl"), ("rotate", 64, "bce")])
def test_host_step_vs_oracle(eng, model, D, loss):
    E, R, n = 3001, 7, 130
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.3)
    tri = orc.make_triples(E, R, n)
    ref = float(orc.train_1vsall_forward(model, ent, rel, tri, loss))
    step = eng.HostStep(model, ent.cuda(), rel.cuda(), n, loss)
    got = step(tri.contiguous().pin_memory())
    assert abs(got - ref) <= 1e-4 * abs(ref), (got, ref)
    assert step.h2d_bytes == n * 24 and step.d2h_bytes == 4


def test_edge_cases(eng):
    ent, rel = orc.make_tables("complex", 100, 3, 32)
    ce, cr = ent.cuda(), rel.cuda()
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    assert eng.score_spo("complex", ce, cr, ce, empty, empty, empty).shape == (0,)
    assert eng.score_1vsN("complex", "sp_", ce, cr, ce, empty, empty).shape == (0, 100)
    one = torch.tensor([5], device="cuda")
    out = eng.score_1vsN("complex", "sp_", ce, cr, ce, one, one % 3, one)
    ref = orc.score_sp("complex", ent, rel, one.cpu(), one.cpu() % 3, one.cpu())
    _assert_close(out, ref, "1x1")
    with pytest.raises(ValueError):
        eng.score_1vsN("complex", "s_o", ce, cr, ce, one, one)
    with pytest.raises(ValueError):  # odd dim
        eng.score_1vsN("complex", "sp_", ce[:, :31].contiguous(), cr, ce[:, :31].contiguous(), one, one)
    with pytest.raises(RuntimeError):  # CPU tensors are refused, never routed to a fallback
        eng.score_1vsN("complex", "sp_", ent, rel, ent, one.cpu(), one.cpu())
    # table widths that are not multiples of 4 floats: no TMA (16-byte alignment) -> scalar SIMT loads
    for model, D in (("complex", 66), ("distmult", 33), ("transe", 35), ("rotate", 70)):
        e2, r2 = orc.make_tables(model, 517, 3, D)
        t2 = orc.make_triples(517, 3, 40)
        got = eng.score_sp_po(model, e2.cuda(), r2.cuda(), t2[:, 0].cuda(), t2[:, 1].cuda(), t2[:, 2].cuda())
        _assert_close(got, orc.score_sp_po(model, e2, r2, t2[:, 0], t2[:, 1], t2[:, 2]), f"{model} D={D}")
        with pytest.raises(NotImplementedError):
            if model in ("transe", "rotate"):
                eng.score_1vsN(model, "sp_", e2.cuda(), r2.cuda(), e2.cuda(), t2[:, 0].cuda(), t2[:, 1].cuda(),
                               precision="3xtf32")
            else:
                eng.score_1vsN(model, "sp_", e2.cuda(), r2.cuda(), e2.cuda(), t2[:, 0].cuda(), t2[:, 1].cuda(),
                               precision="tf32+bf16x2")
    # negative sampling: empty batch, K = 1, duplicate negatives
    tri0 = torch.zeros((0, 3), dtype=torch.int64, device="cuda")
    assert eng.ns_score("complex", ce, cr, tri0, torch.zeros((0, 5), dtype=torch.int64, device="cuda"), 2).shape == (0, 5)
    tri1 = torch.tensor([[1, 2, 3], [4, 0, 5]], device="cuda")
    neg1 = torch.tensor([[7], [7]], device="cuda")
    got = eng.ns_score("complex", ce, cr, tri1, neg1, 0, True)
    ref = orc.ns_scores_with_positive("complex", ent, rel, tri1.cpu(), neg1.cpu(), 0)
    _assert_close(got, ref, "ns K=1")
    # non-contiguous score output rows (ldo > m) and int32 indexes
    big = torch.full((1, 300), -7.0, device="cuda")
    eng.score_1vsN("complex", "sp_", ce, cr, ce, one.int(), (one % 3).int(), out=big[:, :100])
    assert float(big[0, 100]) == -7.0
    _assert_close(big[:, :100], orc.score_sp("complex", ent, rel, one.cpu(), one.cpu() % 3), "strided out")


@pytest.mark.parametrize("model", orc.MODELS)
def test_mid_size_golden(eng, model):
    """The CUDA path against outputs of the LIVE reference at a mid-size shape (E=5003, D=128, n=300; sampled
    columns + row sums, tests/golden/mid_*.npz): closes the chain reference -> oracle -> CUDA at a shape where the
    tensor-core kernels run several K chunks and tiles in both dimensions."""
    import numpy as np
    z = np.load(os.path.join(GOLDEN, f"mid_{model}.npz"))
    E, R, D, n = int(z["E"]), int(z["R"]), int(z["D"]), int(z["n"])
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5, seed=4321)
    tri = orc.make_triples(E, R, n, seed=17).cuda()
    ce, cr = ent.cuda(), rel.cuda()
    s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
    cols = torch.from_numpy(z["cols"])
    x = eng.score_sp_po(model, ce, cr, s, p, o).cpu()
    for got, key in ((x[:, :E], "sp"), (x[:, E:], "po")):
        rms = float(z[key + "_rms"])
        err = float((got[:, cols] - torch.from_numpy(z[key + "_cols"])).abs().max())
        assert err <= TOL * rms, (model, key, err / rms)
        # row sums: every column enters (errors add like sqrt(E) at worst)
        serr = float((got.double().sum(1) - torch.from_numpy(z[key + "_rowsum"])).abs().max())
        assert serr <= TOL * rms * E ** 0.5, (model, key, serr / rms)
    spo = eng.score_spo(model, ce, cr, ce, s, p, o).cpu()
    assert float((spo - torch.from_numpy(z["spo"])).abs().max()) <= TOL * float(z["sp_rms"])
