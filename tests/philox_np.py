"""TEST INFRASTRUCTURE: the embedding-dropout masks of tests/dropout_oracle.py, vectorised over numpy.  Philox4x32-10
runs on uint64 arrays that hold one 32-bit word per lane: M * c < 2^64 for 32-bit M and c, so the high word of a product
is `p >> 32` and the low word `p & 0xFFFFFFFF`.  mask() has the signature and result of dropout_oracle.mask and draws a
[14 541, 512] mask in well under a second, so the fp64 references of the dropout kernels can run at table scale."""
from __future__ import annotations

import numpy as np
import torch

from dropout_oracle import threshold
from philox_ref import M0, M1, MASK, W0, W1

_M0, _M1, _LO = np.uint64(M0), np.uint64(M1), np.uint64(MASK)
_S32 = np.uint64(32)


def philox4x32_10(c0, c1, c2, c3, key):
    """The four output words of Philox4x32-10 for counters (c0, c1, c2, c3) (uint64 arrays or ints of 32-bit words,
    broadcast together) under key = (k0, k1)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in (c0, c1, c2, c3))
    k0, k1 = int(key[0]) & MASK, int(key[1]) & MASK
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = (p1 >> _S32) ^ c1 ^ np.uint64(k0), p1 & _LO, (p0 >> _S32) ^ c3 ^ np.uint64(k1), p0 & _LO
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def mask(p, seed, call, stream, rows, dim, row_base=0):
    """Keep mask [rows, dim] (bool) of draw `stream` over global rows [row_base, row_base + rows): element
    e = row * dim + k takes word e & 3 of the block with counter ((stream << 46) | (e >> 2), call) under key seed."""
    e_lo, e_hi = row_base * dim, (row_base + rows) * dim
    if rows * dim == 0:
        return torch.zeros((rows, dim), dtype=torch.bool)
    g0, g1 = e_lo >> 2, ((e_hi - 1) >> 2) + 1
    hi = np.arange(g0, g1, dtype=np.uint64) | np.uint64(stream << 46)
    w = philox4x32_10(hi & _LO, hi >> _S32, call & MASK, (call >> 32) & MASK, (seed & MASK, (seed >> 32) & MASK))
    words = np.stack(w, 1).reshape(-1)                        # word 4 (g - g0) + j belongs to element 4 g + j
    keep = words[e_lo - 4 * g0:e_hi - 4 * g0] < np.uint64(threshold(p))
    return torch.from_numpy(keep.reshape(rows, dim))
