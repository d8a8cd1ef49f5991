"""The tensor-core scorer's fused BCE epilogue at logit ranges that stress its one-logarithm-per-fragment-row form.

The epilogue sums log(1 + e) over a lane's 32 columns as one log of the product of the factors 1 + e, e = exp(-|z|).
Far from 0 (large table sigma) e underflows and every factor is exactly 1; near 0 (small sigma, with a loss offset)
every factor approaches 2 and a lane's product approaches 2^32.  Each regime runs with full entity tiles and with a
ragged last entity tile (E % 128 != 0), against the fp64 oracle at the suite's 1e-4 relative bar."""
import pytest
import torch

from oracle import kge_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-4

# (sigma, offset): ComplEx D=256 scores have a standard deviation of about 22.6 * sigma^3
REGIMES = {
    "far": (3.0, 0.0),       # |z| ~ 600: e underflows, factors 1
    "near": (0.2, 0.1),      # |z| ~ 0.2: factors near 2, products near 2^32
}


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    return engine


@pytest.mark.parametrize("E", [1024, 1000, 3001], ids=["E1024-full", "E1000-ragged", "E3001-ragged"])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_bce_index_labels_extreme_logits(eng, regime, E):
    sigma, offset = REGIMES[regime]
    model, D, n = "complex", 256, 389
    ent, rel = orc.make_tables(model, E, 11, D, sigma=sigma)
    tri = orc.make_triples(E, 11, n)
    ref = float(orc.train_1vsall_forward(model, ent.double(), rel.double(), tri, "bce", offset))
    got = float(eng.train_1vsall_forward(model, ent.cuda(), rel.cuda(), tri.cuda(), "bce", offset))
    assert abs(got - ref) <= TOL * abs(ref), f"{regime} E={E}: {got} vs {ref}"


@pytest.mark.parametrize("E", [1024, 1000], ids=["E1024-full", "E1000-ragged"])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_bce_dense_labels_extreme_logits(eng, regime, E):
    sigma, offset = REGIMES[regime]
    model, D, n = "complex", 256, 389
    ent, rel = orc.make_tables(model, E, 11, D, sigma=sigma)
    tri = orc.make_triples(E, 11, n)
    g = torch.Generator().manual_seed(E)
    dense = (torch.rand((n, E), generator=g) < 0.01).float()
    scores = orc.score_sp(model, ent.double(), rel.double(), tri[:, 0], tri[:, 1])
    ref = float(orc.bce_loss(scores, dense.double(), offset))
    s, p = tri[:, 0].contiguous().cuda(), tri[:, 1].contiguous().cuda()
    got = float(eng.score_1vsN_loss(model, "sp_", ent.cuda(), rel.cuda(), ent.cuda(), dense.cuda(), s, p, None, "bce",
                                    offset))
    assert abs(got - ref) <= TOL * abs(ref), f"{regime} E={E}: {got} vs {ref}"


def test_bce_near_zero_repeatable(eng):
    """Two identical calls give identical bits with every factor near 2."""
    sigma, offset = REGIMES["near"]
    ent, rel = orc.make_tables("complex", 1000, 11, 256, sigma=sigma)
    tri = orc.make_triples(1000, 11, 389)
    ce, cr, ct = ent.cuda(), rel.cuda(), tri.cuda()
    a = eng.train_1vsall_forward("complex", ce, cr, ct, "bce", offset).item()
    b = eng.train_1vsall_forward("complex", ce, cr, ct, "bce", offset).item()
    assert a == b
