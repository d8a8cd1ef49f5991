"""Parity tests of the gradient kernels (SURVEY 8f-1): the pre-split fp16 GEMM with
split-K accumulation, the analytic backward of the fused 1vsAll step (dot family, BCE and KL) against gradients
of the live reference (tests/golden/grads_*.npz) and against the CPU algebra at medium sizes, and the fused
negative-sampling backward."""
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


def test_gemm_nt_vs_fp64(eng):
    """Pre-split fp16 GEMM (the backward's building block; also exercises presplit + pairwise_tc3 on shapes
    the scorer never sees: long reductions, few rows, K not a multiple of 64, tiny and huge magnitudes)."""
    g = torch.Generator().manual_seed(0)
    for M, N, K, sa, sb in ((300, 500, 1000, 1.0, 1.0), (2048, 512, 14541, 1e-3, 1.0), (130, 40, 72, 50.0, 1e-4),
                            (5000, 384, 2048, 1.0, 1.0)):
        a = torch.randn((M, K), generator=g) * sa
        b = torch.randn((N, K), generator=g) * sb
        ref = a.double() @ b.double().t()
        got = eng.gemm_nt(a.cuda(), b.cuda())
        _assert_close(got, ref, f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("fname", ["grads_complex_bce.npz", "grads_distmult_bce.npz", "grads_simple_bce.npz",
                                   "grads_cp_bce.npz", "grads_rescal_bce.npz", "grads_complex_kl.npz",
                                   "grads_rescal_kl.npz"])
def test_backward_golden(eng, fname):
    """Table gradients of one 1vsAll step (BCE with offset, KL) against the live reference's backward."""
    g = _load(fname)
    model, loss = fname[len("grads_"):-4].split("_")
    d_ent, d_rel = eng.train_1vsall_backward(model, g["ent"].cuda(), g["rel"].cuda(), g["triples"].cuda(), loss,
                                               float(g["offset"]))
    _assert_close(d_ent, g["d_ent"], fname + " d_ent")
    _assert_close(d_rel, g["d_rel"], fname + " d_rel")


@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,D", [("complex", 128), ("distmult", 64), ("simple", 128), ("cp", 64), ("rescal", 24)])
def test_backward_medium(eng, model, D, loss):
    """Ragged medium shapes with duplicate rows, against the analytic CPU assembly (oracle/kge_fold.py, itself
    pinned to autograd and to the reference's gradients)."""
    from oracle import kge_fold as kf

    E, R, n = 3001, 7, 333
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    tri[5] = tri[4]
    off = 0.5 if loss == "bce" else 0.0
    ref_e, ref_r = kf.train_1vsall_backward(model, ent.double(), rel.double(), tri, loss, off)
    d_ent, d_rel = eng.train_1vsall_backward(model, ent.cuda(), rel.cuda(), tri.cuda(), loss, off)
    _assert_close(d_ent, ref_e, f"{model} d_ent")
    _assert_close(d_rel, ref_r, f"{model} d_rel")


@pytest.mark.parametrize("loss", ["bce", "kl"])
@pytest.mark.parametrize("model,D,ln", [("transe", 100, 1.0), ("transe", 72, 2.0), ("rotate", 72, 1.0), ("transe", 3, 1.0),
                                        ("transe", 130, 2.0), ("rotate", 66, 1.0)])
def test_backward_distance_family(eng, model, D, ln, loss):
    """The 1vsAll backward of TransE (L1, L2) and RotatE (L1): CUDA-core scores, dense G and the two row-gradient passes
    of grad_distance.cu, against the analytic CPU assembly; ragged sizes (E, 2n not multiples of the 128 / 16 tiles, D not
    a multiple of the 64-element chunk) and a duplicate triple."""
    from oracle import kge_fold as kf

    E, R, n = 1201, 7, 139
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    tri[5] = tri[4]
    off = 0.5 if loss == "bce" else 0.0
    ref_e, ref_r = kf.train_1vsall_backward(model, ent.double(), rel.double(), tri, loss, off, ln)
    d_ent, d_rel = eng.train_1vsall_backward(model, ent.cuda(), rel.cuda(), tri.cuda(), loss, off, ln)
    _assert_close(d_ent, ref_e, f"{model} d_ent")
    _assert_close(d_rel, ref_r, f"{model} d_rel")


def test_backward_distance_family_tiny_batch(eng):
    """One triple, five entities: every tile of the row-gradient passes is ragged."""
    from oracle import kge_fold as kf

    ent, rel = orc.make_tables("transe", 5, 2, 8, sigma=0.5)
    tri = torch.tensor([[1, 0, 3]])
    ref_e, ref_r = kf.train_1vsall_backward("transe", ent.double(), rel.double(), tri, "kl", 0.0, 1.0)
    d_ent, d_rel = eng.train_1vsall_backward("transe", ent.cuda(), rel.cuda(), tri.cuda(), "kl", 0.0, 1.0)
    _assert_close(d_ent, ref_e, "d_ent")
    _assert_close(d_rel, ref_r, "d_rel")


def test_backward_distance_family_refuses_other_norms(eng):
    ent, rel = orc.make_tables("rotate", 50, 3, 16, sigma=0.5)
    tri = orc.make_triples(50, 3, 8)
    with pytest.raises(NotImplementedError):
        eng.train_1vsall_backward("rotate", ent.cuda(), rel.cuda(), tri.cuda(), "bce", 0.0, 2.0)


@pytest.mark.parametrize("model,D,ln", [("complex", 64, 1.0), ("distmult", 32, 1.0), ("simple", 64, 1.0), ("cp", 64, 1.0),
                                        ("rescal", 16, 1.0), ("transe", 64, 1.0), ("transe", 64, 2.0), ("rotate", 64, 1.0)])
def test_ns_backward(eng, model, D, ln):
    """Fused negative-sampling backward (S and O slots, positive column included) against the CPU algebra
    (oracle/kge_fold.ns_backward, itself pinned to the reference job's gradients)."""
    from oracle import kge_fold as kf

    E, R, n, K = 501, 5, 37, 150
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    g = torch.Generator().manual_seed(3)
    negs = {S: torch.randint(0, E, (n, K), generator=g), O: torch.randint(0, E, (n, K + 7), generator=g)}
    ref_e, ref_r = kf.ns_backward(model, ent.double(), rel.double(), tri, negs, 0.25, ln)
    d_ent, d_rel = eng.ns_backward(model, ent.cuda(), rel.cuda(), tri.cuda(), {k: v.cuda() for k, v in negs.items()},
                                     0.25, ln)
    _assert_close(d_ent, ref_e, f"{model} d_ent")
    _assert_close(d_rel, ref_r, f"{model} d_rel")


@pytest.mark.parametrize("model,D,ln", [("complex", 128, 1.0), ("distmult", 64, 1.0), ("simple", 128, 1.0), ("cp", 64, 1.0),
                                        ("rescal", 24, 1.0), ("transe", 72, 1.0), ("transe", 72, 2.0), ("rotate", 72, 1.0)])
@pytest.mark.parametrize("combine", ["sp_", "_po"])
def test_score_1vsN_backward_vs_autograd(eng, model, D, ln, combine):
    """Backward of a dense [n, E] score block given dL/dscores (the unfused route of a job: score_sp -> KgeLoss ->
    autograd) against torch autograd of the oracle's expression in fp64."""
    E, R, n = 3001, 5, 150
    ent, rel = orc.make_tables(model, E, R, D, sigma=0.5)
    tri = orc.make_triples(E, R, n)
    q = tri[:, 0] if combine == "sp_" else tri[:, 2]
    g = torch.randn((n, E), generator=torch.Generator().manual_seed(2)) * 0.1
    e64, r64 = ent.double().requires_grad_(True), rel.double().requires_grad_(True)
    if combine == "sp_":
        x = orc.score_emb(model, e64[q], r64[tri[:, 1]], e64, "sp_", ln)
    else:
        x = orc.score_emb(model, e64, r64[tri[:, 1]], e64[q], "_po", ln)
    ref_e, ref_r = torch.autograd.grad(x, (e64, r64), g.double())
    d_ent, d_rel = eng.score_1vsN_backward(model, combine, ent.cuda(), rel.cuda(), q.cuda(), tri[:, 1].cuda(), g.cuda(), ln)
    _assert_close(d_ent, ref_e, f"{model} {combine} d_ent")
    _assert_close(d_rel, ref_r, f"{model} {combine} d_rel")
