"""TEST INFRASTRUCTURE: fp64 per-row terms of the fused 1vsAll / KvsAll losses and the rounding bound a kernel row
must meet when it is compared with the fp64 loss of the kernel's OWN fp32 scores.

The engine's store form and fused-loss forms of one batch run the same scoring arithmetic (capi.cu, run_block), so the
scores a loss epilogue saw can be read back through score_1vsN / score_sp_po.  Comparing each kernel row with the fp64
loss of those scores isolates the epilogue, the slot scheme and the finaliser from the scoring error: the bar is a
rounding bound of the row's own fp32 reduction, not a fraction of the batch total.

Labels come in the forms the engine takes: a 1-D index tensor (-1: the row has no label), a dense [n, E] matrix, or a
CSR pair (offsets, cols) whose labels are y = (1 - eps) * count + (eps > 0 ? 1/E : 0)  (train_KvsAll.py:242-266).

Row bound   |kernel_i - fp64_i| <= C * u * d_i * M_i,   u = 2^-24, C = 4

d_i is the depth of the fp32 computation the kernel performs for row i: the largest number of roundings between one
score and the row loss (see tc_depth / simt_depth / dense_depth; k = 1 rounding per accumulation step for BCE, 2 for
KL, whose online log-sum-exp rescales (multiply) and adds at every step).  M_i is the row's magnitude:

  BCE   M_i = sum_j softplus(x_ij) + sum_j |y_ij x_ij| + N_i              x = z + offset
  KL    M_i = 1 + |lse_i| + ln E + |ln yc_i| + (sum_j |y_ij z_ij| + sum_j |y_ij ln y_ij|) / yc_i
        (CSR form: + |z_i0|)                                              yc = max(sum_j y_ij, 1e-12)

Derivation.  A sum evaluated by any tree whose leaves pass through at most d roundings is within gamma_d * sum |t_j|
(gamma_d = d u / (1 - d u) < 1.01 d u here) of the exact sum of its terms (Higham, Accuracy and Stability of Numerical
Algorithms, 4.2).  The rest is the error of the terms themselves, each shown to be at most 4 u d_i times its share of
M_i (every d_i below is >= 20, and >= 44 on the tensor-core path):

BCE (tc_common.cuh:146-166 tensor core, common.cuh:153-162 / 265-272 CUDA core and dense, epilogue_dense.cu:74-82):
  * x = v + off rounds once: u |x| per score, <= u softplus(x) in max(x, 0) and <= u |y x| in the label term.
  * e = exp(-|x|) by ex2.approx (PTX ISA: at most 2 ulp, 4 u relative) of -|x| * LOG2E, whose rounding and that of
    the constant shift the exponent by 2 u |x| log2(e): relative error (4 + 2 |x|) u in e.  Since
    log(1 + e) >= e ln 2, that is <= (6 + 3 |x|) u of the term log(1 + e) <= softplus(x): within 4 u d softplus(x)
    for |x| <= 4 d / 3 - 2 (>= 56 here), and beyond that e < 1e-24, far below anything else in the bound.
  * Tensor core, one logarithm per lane and tile (tc_common.cuh:156): the product of up to 32 factors 1 + e rounds
    63 times (u relative each, 63 u absolute after the logarithm), lg2.approx adds <= 2^-22.6 (2.7 u) absolute
    before the ln 2 scaling: <= 66 u per logarithm, N_i of them (tc_log_count).  4 u d_i >= 176 u covers it.
  * CUDA core / dense (softplus_f): __logf(1 + e) is lg2.approx again (<= 3 u absolute with the rounding of 1 + e)
    for every score whose e >= 1e-5; N_i counts the scores with |x| < 30 (log_count), which covers those and the
    absolute error 2 u |x| e of the rest.  The label term y * x is one fma per score.
  * row = a - b rounds once more (counted in d).
KL (tc_common.cuh:168-198, common.cuh:181-191 / 273-287, epilogue_dense.cu:83-98):
  * every exponential exp(v - mn) and every rescale exp(m_old - mn) is ex2.approx of an argument formed with the
    rounded LOG2E and mn * LOG2E: relative error 4 u + u |mn| + 2 u |v - mn| per factor.  Along the path of score j
    the shifts (v - mn) and (m_old - mn) add up to at most m - z_j, and sum_j p_j (m - z_j) <= sum_j p_j (lse - z_j)
    = H(p) <= ln E (p = softmax(z)).  With |m| <= |lse| + ln E the relative error of s is within
    u (k d + |lse| + 3 ln E + 4), which logf turns into an absolute error of lse: covered by 1 + |lse| + ln E.
  * lse = m + logf(s), its rounding u |lse|.  w = y_sum / yc is exactly 1 (or 0).
  * y_sum carries a relative error <= d u (positive terms), which moves ylogy / yc and yx / yc by that relative
    amount and ln yc by d u absolute (the 1); logf(yc) rounds by u |ln yc|.  yx is a sum of |y z| terms.
  * y ln y uses __logf (<= 2^-21.4 absolute, 6 u, or 2 ulp relative): <= 6 u y + 4 u |y ln y| per label, i.e.
    6 u (sum y / yc = 1) + 4 u sum |y ln y| / yc after the division.
  * CSR form (csr_loss.cu:78-82): lse is rebuilt as (lse - z_i0) + z_i0, two more roundings of at most
    u (|lse| + |z_i0|).
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
C = 4.0

TC_TILE = 128            # pairwise_tc.cu TM = TN
SIMT_TILE = 128          # pairwise_simt.cu BN = BM
SIMT_CHUNK_CTAS = 132 * 6   # pairwise_simt_nchunks
DENSE_CHUNK, DENSE_THREADS = 4096, 256   # epilogue_dense.cu DN_CHUNK, DN_THREADS


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


# --------------------------------------------------------------------------- labels and fp64 rows
def dense_labels(labels, n: int, E: int, smoothing: float = 0.0, dtype=torch.float64, device=None) -> torch.Tensor:
    """The [n, E] label matrix of index, dense or CSR (offsets, cols) labels; smoothing applies to CSR labels as the
    engine applies it (y = (1 - eps) * count + 1/E)."""
    if isinstance(labels, (tuple, list)):
        offs, cols = labels
        dev = device if device is not None else cols.device
        counts = (offs[1:] - offs[:-1]).to(dev)
        rows = torch.repeat_interleave(torch.arange(n, device=dev), counts)
        y = torch.zeros((n, E), dtype=dtype, device=dev)
        y.index_put_((rows, cols.to(dev).long()), torch.ones(rows.numel(), dtype=dtype, device=dev), accumulate=True)
        if smoothing > 0.0:
            y = (1.0 - smoothing) * y + 1.0 / E
        return y
    if labels.dim() == 2:
        return labels.to(dtype=dtype, device=device if device is not None else labels.device)
    dev = device if device is not None else labels.device
    idx = labels.to(dev).long()
    y = torch.zeros((n, E), dtype=dtype, device=dev)
    has = idx >= 0
    y[torch.arange(n, device=dev)[has], idx[has]] = 1.0
    return y


def bce_rows(z: torch.Tensor, labels, offset: float = 0.0, smoothing: float = 0.0) -> torch.Tensor:
    """Row i of BCEWithLogitsKgeLoss (sum):  sum_j softplus(z_ij + off) - sum_j y_ij (z_ij + off), in fp64."""
    x = z.double() + offset
    y = dense_labels(labels, x.shape[0], x.shape[1], smoothing, device=x.device)
    sp = torch.clamp(x, min=0.0) + torch.log1p(torch.exp(-x.abs()))
    return sp.sum(1) - (y * x).sum(1)


def kl_rows(z: torch.Tensor, labels, smoothing: float = 0.0) -> torch.Tensor:
    """Row i of KLDivWithSoftmaxKgeLoss (sum): KLDiv(log_softmax(z_i), y_i / max(sum y_i, 1e-12)), in fp64; 0 for a
    row without label mass.  With index labels this is the cross entropy lse_i - z_i,label."""
    x = z.double()
    y = dense_labels(labels, x.shape[0], x.shape[1], smoothing, device=x.device)
    t = y / torch.clamp(y.sum(1, keepdim=True), min=1e-12)
    return (torch.xlogy(t, t) - t * torch.log_softmax(x, 1)).sum(1)


def loss_rows(loss: str, z, labels, offset: float = 0.0, smoothing: float = 0.0) -> torch.Tensor:
    return bce_rows(z, labels, offset, smoothing) if loss == "bce" else kl_rows(z, labels, smoothing)


# --------------------------------------------------------------------------- reduction depths
def tc_schedule(nq: int, m: int, sms: int):
    """pairwise_tc.cu schedule(): (q_tiles, e_tiles, items, grid, nchunks = 2 * nsl)."""
    q_tiles = max(1, _cdiv(nq, TC_TILE))
    e_tiles = _cdiv(m, TC_TILE)
    items = q_tiles * e_tiles
    grid = min(items, sms)
    per = items // grid
    nsl = min(_cdiv(e_tiles, per) + 1, grid)
    return q_tiles, e_tiles, items, grid, 2 * nsl


def tc_tiles_per_slot(nq: int, m: int, sms: int, ping_pong: bool):
    """Per query tile, the most entity tiles whose states one slot accumulates (pairwise_tc.cu:224-340): a CTA covers
    the items [b * items / grid, (b + 1) * items / grid); ping-pong warpgroup g takes the items i with (i - i0) % 2 == g,
    the row-split warpgroups take all of them."""
    q_tiles, e_tiles, items, grid, _ = tc_schedule(nq, m, sms)
    out = [0] * q_tiles
    for b in range(grid):
        i0, i1 = b * items // grid, (b + 1) * items // grid
        for qt in range(i0 // e_tiles, (i1 - 1) // e_tiles + 1):
            lo, hi = max(i0, qt * e_tiles), min(i1, (qt + 1) * e_tiles)
            cnt = hi - lo
            if ping_pong:
                even = _cdiv(hi - i0, 2) - _cdiv(lo - i0, 2)
                cnt = max(even, cnt - even)
            out[qt] = max(out[qt], cnt)
    return out


def _fin_depth(k: int, nchunks: int) -> int:
    # loss_finalize_kernel: ceil(nchunks / 32) slots per lane in order, a 5-level shuffle tree, then the row formula
    return k * _cdiv(nchunks, 32) + 5 * k + 3


def tc_depth(loss: str, nq: int, m: int, sms: int, ping_pong: bool = True) -> torch.Tensor:
    """d_i of the tensor-core epilogue: 32 scores per lane and tile, 2 roundings per tile folded into the lane's state,
    the quad's lane reduction (4 lanes ping-pong, 2 row-split), then the finaliser over 2 * nsl slots."""
    k = 1 if loss == "bce" else 2
    nch = tc_schedule(nq, m, sms)[4]
    lanes = 4 if ping_pong else 2
    per_qt = [32 + 2 * t + k * int(math.log2(lanes)) + _fin_depth(k, nch)
              for t in tc_tiles_per_slot(nq, m, sms, ping_pong)]
    return torch.tensor(per_qt, dtype=torch.float64).repeat_interleave(TC_TILE)[:nq]


def simt_nchunks(nq: int, m: int) -> int:
    """pairwise_simt_nchunks."""
    ct, rt = _cdiv(m, SIMT_TILE), _cdiv(nq, SIMT_TILE)
    return min(max(1, (SIMT_CHUNK_CTAS + rt - 1) // max(rt, 1)), ct)


def simt_depth(loss: str, nq: int, m: int) -> torch.Tensor:
    """d_i of the CUDA-core epilogue: a thread's 8 columns per tile over its chunk's tiles, one (BCE) or two (KL)
    roundings each, a 16-lane reduction, then the finaliser over the chunks."""
    k = 1 if loss == "bce" else 2
    nch = simt_nchunks(nq, m)
    tiles = _cdiv(_cdiv(m, SIMT_TILE), nch)
    return torch.full((nq,), float(k * 8 * tiles + 4 * k + _fin_depth(k, nch)), dtype=torch.float64)


def dense_depth(loss: str, nq: int, m: int) -> torch.Tensor:
    """d_i of dense_epilogue_kernel: a thread's <= 16 columns of a 4096-column chunk, the block's 8-level reduction,
    then the finaliser over the chunks."""
    k = 1 if loss == "bce" else 2
    per = _cdiv(min(m, DENSE_CHUNK), DENSE_THREADS)
    return torch.full((nq,), float(k * per + 8 * k + _fin_depth(k, _cdiv(m, DENSE_CHUNK))), dtype=torch.float64)


def csr_extra_depth(offs: torch.Tensor) -> torch.Tensor:
    """csr_rows_kernel: a row's listed scores strided over 32 lanes, a 5-level shuffle, and the row formula."""
    nnz = (offs[1:] - offs[:-1]).double().cpu()
    return torch.ceil(nnz / 32) + 5 + 4


def tc_log_count(nq: int, m: int) -> torch.Tensor:
    """N_i on the tensor-core path: one logarithm per lane of the quad and entity tile that holds a valid column (lane q
    holds columns 2q + 8j (+1) of the tile, tc_common.cuh:277)."""
    e_tiles = _cdiv(m, TC_TILE)
    r = m - TC_TILE * (e_tiles - 1)
    return torch.full((nq,), float(4 * (e_tiles - 1) + min(4, _cdiv(r, 2))), dtype=torch.float64)


def log_count(z: torch.Tensor, offset: float = 0.0) -> torch.Tensor:
    """N_i on the CUDA-core and dense paths: the scores with |z + off| < 30."""
    return ((z.double() + offset).abs() < 30.0).sum(1).double()


# --------------------------------------------------------------------------- the bound
def row_bound(loss: str, z: torch.Tensor, labels, depth, offset: float = 0.0, n_log=None, smoothing: float = 0.0,
              csr: bool = False) -> torch.Tensor:
    """C u d_i M_i for every row (module docstring).  depth: [n] (or scalar) d_i; n_log: [n] N_i (BCE)."""
    x = z.double()
    n, E = x.shape
    y = dense_labels(labels, n, E, smoothing, device=x.device)
    d = torch.as_tensor(depth, dtype=torch.float64).to(x.device)
    if loss == "bce":
        xo = x + offset
        sp = torch.clamp(xo, min=0.0) + torch.log1p(torch.exp(-xo.abs()))
        M = sp.sum(1) + (y * xo).abs().sum(1)
        if n_log is not None:
            M = M + torch.as_tensor(n_log, dtype=torch.float64).to(x.device)
    else:
        lse = torch.logsumexp(x, 1)
        yc = torch.clamp(y.sum(1), min=1e-12)
        lab = ((y * x).abs().sum(1) + torch.xlogy(y, y).abs().sum(1)) / yc
        M = 1.0 + lse.abs() + math.log(E) + torch.log(yc).abs() + lab
        if csr:
            M = M + x[:, 0].abs()
    return C * U * d * M
