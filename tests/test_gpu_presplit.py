"""Parity tests of the default tensor-core path: operands pre-split into row-scaled fp16 hi/lo planes
(presplit.cu) scored by pairwise_tc.cu (AUTO / precision "f16x3").  Bar: floating point <= 1e-4 * rms, rank/tie
counts bit-exact on the kernel's own scores."""
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

    assert torch.cuda.is_available() and engine.device_ok()
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


def test_presplit_fp16_golden(eng):
    for fname, model in (("scores_complex.npz", "complex"), ("scores_distmult.npz", "distmult"),
                         ("scores_simple.npz", "simple"), ("scores_complex_sigma01.npz", "complex")):
        g = _load(fname)
        ent, rel, tri = g["ent"].cuda(), g["rel"].cuda(), g["triples"].cuda()
        s, p, o = tri[:, S].contiguous(), tri[:, P].contiguous(), tri[:, O].contiguous()
        sub = g["subset"].cuda()
        for prec in ("auto", "f16x3"):
            _assert_close(eng.score_1vsN(model, "sp_", ent, rel, ent, s, p, None, precision=prec), g["sp"], fname + " sp")
            _assert_close(eng.score_1vsN(model, "_po", ent, rel, ent, o, p, sub, precision=prec), g["po_subset"], fname + " po_subset")
            _assert_close(eng.score_sp_po(model, ent, rel, s, p, o, None, precision=prec), g["sp_po"], fname + " sp_po")


@pytest.mark.parametrize("sigma", [1.0, 1e-3])
def test_presplit_fp16_medium(eng, sigma):
    """Dense scores, gathered candidate subsets, fused BCE/KL, fused rank counting at ragged sizes (tiles cut in
    both dimensions, K not a multiple of the 64-wide chunk for RESCAL/CP), including tiny-valued tables that a
    fixed fp16 scale would flush."""
    for model, D in (("complex", 192), ("distmult", 64), ("simple", 128), ("rescal", 40), ("cp", 200)):
        E, R, n = 6007, 7, 389
        ent, rel = orc.make_tables(model, E, R, D, sigma=sigma)
        tri = orc.make_triples(E, R, n)
        ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
        s, p, o = ct[:, S].contiguous(), ct[:, P].contiguous(), ct[:, O].contiguous()
        ref = orc.score_sp_po(model, ent, rel, tri[:, S], tri[:, P], tri[:, O])
        _assert_close(eng.score_sp_po(model, ce, cr, s, p, o), ref, f"{model} sp_po")
        sub = torch.randperm(E, generator=torch.Generator().manual_seed(1))[:1500]
        got = eng.score_1vsN(model, "_po", ce, cr, ce, o, p, sub.cuda())
        _assert_close(got, orc.score_po(model, ent, rel, tri[:, P], tri[:, O], sub), f"{model} po subset")
        if model == "cp":
            continue        # stacked fused epilogues are not offered for CP
        for loss in ("bce", "kl"):
            refl = float(orc.train_1vsall_forward(model, ent, rel, tri, loss))
            gotl = float(eng.train_1vsall_forward(model, ce, cr, ct, loss))
            assert abs(gotl - refl) <= 1e-4 * abs(refl), (model, loss, gotl, refl)
        dense = eng.score_1vsN(model, "sp_", ce, cr, ce, s, p)
        true = dense[torch.arange(n, device="cuda"), o].clone()
        rr, tt = orc.ranks_and_ties(dense.cpu(), true.cpu())
        r, t = eng.score_1vsN_rank(model, "sp_", ce, cr, ce, true, s, p)
        assert torch.equal(r.cpu(), rr) and torch.equal(t.cpu(), tt)


def test_presplit_fp16_headline_shape(eng):
    """BASELINE configs[1] shape: the loss repeats to 1e-5 and the scores match the oracle."""
    E, R, D, n = 14541, 237, 512, 1024
    ent, rel = orc.make_tables("complex", E, R, D)
    tri = orc.make_triples(E, R, n)
    ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
    base = float(eng.train_1vsall_forward("complex", ce, cr, ct, "bce"))
    got = float(eng.train_1vsall_forward("complex", ce, cr, ct, "bce"))
    assert abs(got - base) <= 1e-5 * abs(base), (got, base)
    ref = orc.score_sp("complex", ent, rel, tri[:64, S], tri[:64, P])
    _assert_close(eng.score_1vsN("complex", "sp_", ce, cr, ce, ct[:64, S].contiguous(), ct[:64, P].contiguous()), ref,
                  "headline sp")
