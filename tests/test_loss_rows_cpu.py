"""The fp64 per-row losses and their rounding bound (tests/loss_rows_oracle.py), without a GPU.

The rows must add up to the oracle's batch losses for every label form; the bound must hold for honest fp32 evaluations
of the same rows, including one that sums sequentially over E; and it must be tight enough that one dropped label term,
one dropped 128-column chunk or one duplicated chunk of a row exceeds it at the tensor-core path's depth."""
import numpy as np
import pytest
import torch

import loss_rows_oracle as lr
from oracle import kge_oracle as orc

N, E = 64, 3001
SMS = 132    # H100 SXM


def _scores(seed, sigma=1.0, n=N, m=E):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((n, m), generator=g) * sigma).float()


def _labels(kind, n=N, m=E, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "index":
        return torch.randint(0, m, (n,), generator=g)
    dense = (torch.rand((n, m), generator=g) < 0.01).float()
    dense[torch.arange(n), torch.randint(0, m, (n,), generator=g)] = 1.0
    if kind == "dense":
        return dense
    offs = torch.zeros(n + 1, dtype=torch.int64)
    offs[1:] = dense.sum(1).long().cumsum(0)
    return offs, dense.nonzero()[:, 1].contiguous()


@pytest.mark.parametrize("kind", ["index", "dense", "csr-smoothed"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_rows_sum_to_oracle_loss(loss, kind):
    z = _scores(1).double()
    labels = _labels(kind.split("-")[0])
    eps = 0.1 if kind == "csr-smoothed" else 0.0
    rows = lr.loss_rows(loss, z, labels, offset=0.3 if loss == "bce" else 0.0, smoothing=eps)
    y = lr.dense_labels(labels, N, E, eps) if kind != "index" else labels
    if kind == "csr-smoothed":
        assert torch.allclose(y, orc.kvsall_smooth_labels(lr.dense_labels(labels, N, E), eps))
    ref = orc.bce_loss(z, y, 0.3) if loss == "bce" else orc.kl_loss(z, y)
    assert abs(float(rows.sum()) - float(ref)) <= 1e-12 * abs(float(ref))


def test_index_rows_closed_forms():
    z = _scores(2).double()
    lab = _labels("index")
    lab[3] = -1
    kl = lr.kl_rows(z, lab)
    assert float(kl[3]) == 0.0
    lse = torch.logsumexp(z, 1)
    keep = torch.arange(N) != 3
    assert torch.allclose(kl[keep], (lse - z[torch.arange(N), lab.clamp(min=0)])[keep], rtol=1e-13, atol=0)
    zero = torch.zeros((2, E), dtype=torch.float64)
    assert torch.allclose(lr.kl_rows(zero, torch.tensor([0, E - 1])), torch.full((2,), np.log(E), dtype=torch.float64))
    b = lr.bce_rows(zero, torch.tensor([0, -1]), offset=0.25)
    sp = E * float(np.logaddexp(0.0, 0.25))
    assert torch.allclose(b, torch.tensor([sp - 0.25, sp], dtype=torch.float64), rtol=1e-13, atol=0)


# --------------------------------------------------------------------------- honest fp32 evaluations
def _fp32_rows(loss, z, y, offset, chunk):
    """The rows in fp32: terms in fp32, summed sequentially within chunks of `chunk` columns and then sequentially
    over the chunks (chunk = E: one sequential pass over the row).  Returns the rows and their depth."""
    z = z.numpy().astype(np.float32)
    y = y.numpy().astype(np.float32)
    n, m = z.shape

    def seq(t):         # sequential fp32 sums within chunks, then over the chunks
        parts = [np.cumsum(t[:, c:c + chunk], axis=1, dtype=np.float32)[:, -1] for c in range(0, m, chunk)]
        return np.cumsum(np.stack(parts, 1), axis=1, dtype=np.float32)[:, -1]
    depth = min(chunk, m) + lr._cdiv(m, chunk) + 3
    if loss == "bce":
        x = (z + np.float32(offset)).astype(np.float32)
        sp = (np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))).astype(np.float32)
        return (seq(sp) - seq((y * x).astype(np.float32))).astype(np.float32), depth
    mx = z.max(1, keepdims=True)
    s = seq(np.exp(z - mx).astype(np.float32))
    lse = (mx[:, 0] + np.log(s)).astype(np.float32)
    ys = seq(y)
    yc = np.maximum(ys, np.float32(1e-12))
    with np.errstate(divide="ignore", invalid="ignore"):
        ylogy = seq(np.where(y > 0, y * np.log(np.where(y > 0, y, 1)), 0).astype(np.float32))
    yx = seq((y * z).astype(np.float32))
    rows = np.where(ys > 0, ylogy / yc - np.log(yc) - yx / yc + lse, 0).astype(np.float32)
    return rows, 2 * depth


@pytest.mark.parametrize("chunk", [128, E], ids=["chunked", "sequential"])
@pytest.mark.parametrize("case", ["index", "dense", "smoothed", "near-zero", "far"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_bound_holds_for_fp32_evaluation(loss, case, chunk):
    sigma, offset = {"near-zero": (0.2, 0.1), "far": (40.0, 0.5)}.get(case, (3.0, 0.3))
    z = _scores(3, sigma)
    labels = _labels("index" if case in ("index", "near-zero", "far") else "dense", seed=4)
    y = lr.dense_labels(labels, N, E, dtype=torch.float32)
    if case == "smoothed":
        y = orc.kvsall_smooth_labels(y, 0.1)
    off = offset if loss == "bce" else 0.0
    rows, depth = _fp32_rows(loss, z, y, off, chunk)
    ref = lr.loss_rows(loss, z, y.double(), off)
    bound = lr.row_bound(loss, z, y.double(), depth, off)
    ratio = (torch.from_numpy(rows).double() - ref).abs() / bound
    i = int(ratio.argmax())
    assert float(ratio[i]) <= 1.0, f"row {i}: ratio {float(ratio[i]):.3f}"


# --------------------------------------------------------------------------- the bound catches single-row faults
def _tc_bound(loss, z, labels):
    d = lr.tc_depth(loss, N, E, SMS)
    n_log = lr.tc_log_count(N, E) if loss == "bce" else None
    return lr.row_bound(loss, z, labels, d, 0.0, n_log)


def _faulty(loss, z, y, row, cols, dup=False):
    """Row `row` recomputed as a kernel would if it lost (or counted twice) the columns `cols`."""
    keep = torch.ones(z.shape[1], dtype=torch.bool)
    keep[cols] = False
    zr, yr = z[row:row + 1], y[row:row + 1]
    if dup:
        zr, yr = torch.cat([zr, zr[:, cols]], 1), torch.cat([yr, yr[:, cols]], 1)
    else:
        zr, yr = zr[:, keep], yr[:, keep]
    return float(lr.loss_rows(loss, zr, yr)[0])


@pytest.mark.parametrize("kind", ["index", "dense"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_bound_catches_dropped_label_term(loss, kind):
    """A label term of size 0.5 (scores of rms 1) that the epilogue misses."""
    z = _scores(5).double()
    labels = _labels(kind, seed=6)
    y = lr.dense_labels(labels, N, E)
    row = 7
    col = int(y[row].nonzero()[0])
    z[row, col] = 0.5
    ref = lr.loss_rows(loss, z, y)
    bound = _tc_bound(loss, z, y)
    y2 = y.clone()
    y2[row, col] = 0.0
    bad = float(lr.loss_rows(loss, z, y2)[row])
    assert abs(bad - float(ref[row])) > float(bound[row]), (bad, float(ref[row]), float(bound[row]))


@pytest.mark.parametrize("dup", [False, True], ids=["dropped", "duplicated"])
@pytest.mark.parametrize("start", [0, 2816], ids=["first-chunk", "last-full-chunk"])
@pytest.mark.parametrize("loss", ["bce", "kl"])
def test_bound_catches_128_column_chunk(loss, start, dup):
    z = _scores(8).double()
    y = lr.dense_labels(_labels("index", seed=9), N, E)
    ref = lr.loss_rows(loss, z, y)
    bound = _tc_bound(loss, z, y)
    row = 11
    bad = _faulty(loss, z, y, row, list(range(start, start + 128)), dup)
    assert abs(bad - float(ref[row])) > float(bound[row]), (bad, float(ref[row]), float(bound[row]))


def test_bound_is_not_loose():
    """At the tensor-core depth the bound stays a small fraction of a label term that a 1e-4 bar on the batch total
    hides: a KL row of rms-1 scores is bounded well below 1e-3, a BCE row well below 0.1."""
    z = _scores(10).double()
    y = lr.dense_labels(_labels("index", seed=11), N, E)
    assert float(_tc_bound("kl", z, y).max()) < 1e-3
    assert float(_tc_bound("bce", z, y).max()) < 0.1


def test_tc_schedule_matches_kernel_rules():
    # 7 x 47 tiles over 132 CTAs: ranges of 2 and 3 items, ping-pong halves of 1 or 2 tiles
    q_tiles, e_tiles, items, grid, nch = lr.tc_schedule(389, 6007, SMS)
    assert (q_tiles, e_tiles, items, grid) == (4, 47, 188, 132)
    assert nch == 2 * min(47 + 1, 132)
    t = lr.tc_tiles_per_slot(389, 6007, SMS, True)
    assert max(t) == 1 and len(t) == 4
    assert lr.tc_tiles_per_slot(389, 6007, SMS, False) == [2, 2, 2, 2]
    # one query tile against 196 entity tiles: 132 CTAs of 1 or 2 items
    assert lr.tc_schedule(32, 25000, SMS)[4] == 2 * 132
    assert lr.tc_log_count(1, 1025)[0] == 4 * 8 + 1
