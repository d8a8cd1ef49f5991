"""TEST INFRASTRUCTURE: b200kge_sample_frequency and b200kge_sample_frequency_filtered (kge_b200/csrc/rowwise.cu)
restated on numpy, vectorised over the elements of a call, the weights of b200kge_frequency_cdf_build restated on Python
integers, and the definition the entries implement, element by element on the plain-Python Philox.

Weights: q_x = round((c_x + alpha) * 2^s), half to even, s >= 0 the largest integer with Q = sum q_x <= 2^62; cdf is
their exclusive prefix.  Element e = i*K + k takes the word r of b200kge_sample_uniform (pair e & 1 of Philox block
(e // 2, offset) under key seed), t = floor(r * Q / 2^64), x = the largest id with cdf[x] <= t.  Filtered: if x is a
positive of row i's key, u = floor(r' * (Q - M) / 2^64) with r' the same pair of block (e // 2 | 2^63, offset) and M the
weight of the key's positives, and the output is the id holding the u-th unit of non-positive weight.  Absent keys are
unfiltered; rows with Q - M = 0 get -1."""
from __future__ import annotations

import bisect
import math

import numpy as np

import ns_filter_oracle as nfo
import philox_ref

LIMIT = 1 << 62


def _quantised(counts, alpha, s):
    qa = round(math.ldexp(alpha, s))                    # alpha * 2^s is exact; round() is half to even
    return [(int(c) << s) + qa for c in counts]


def quantise(counts, alpha):
    """q as a list of Python ints, and s."""
    counts = [int(c) for c in counts]
    w = sum(counts) + alpha * len(counts)
    if w <= 0:
        raise ValueError("all weights are zero")
    s = max(0, 62 - math.ceil(math.log2(w)) + 2)
    while sum(_quantised(counts, alpha, s)) > LIMIT:
        s -= 1
    if s < 0:
        raise ValueError("the smoothed counts sum to more than 2^62")
    return _quantised(counts, alpha, s), s


def cdf_of(q):
    """The exclusive prefix [V+1] of q, uint64."""
    return np.concatenate([[0], np.cumsum(np.asarray(q, dtype=np.uint64), dtype=np.uint64)]).astype(np.uint64)


def search(cdf, t):
    """The largest x with cdf[x] <= t, for each t (cdf[0] <= t < cdf[-1])."""
    return np.searchsorted(np.asarray(cdf, dtype=np.uint64), np.asarray(t, dtype=np.uint64), side="right") - 1


def below_of(cdf, offsets, values):
    """G [nnz] uint64: for every value v_j of a key, cdf[v_j] minus the weight of the key's values before it."""
    cdf = np.asarray(cdf, dtype=np.uint64)
    offsets, values = np.asarray(offsets, dtype=np.int64), np.asarray(values, dtype=np.int64)
    q = cdf[values + 1] - cdf[values]
    G = np.empty(len(values), dtype=np.uint64)
    for k in range(len(offsets) - 1):
        a, b = offsets[k] - offsets[0], offsets[k + 1] - offsets[0]
        before = np.concatenate([[0], np.cumsum(q[a:b], dtype=np.uint64)[:-1]]).astype(np.uint64)
        G[a:b] = cdf[values[a:b]] - before
    return G


def rest_of(cdf, v, G):
    """Q - M: the weight of the non-positives of a key with positives v (ascending) and below-table G."""
    cdf = np.asarray(cdf, dtype=np.uint64)
    return cdf[-1] - (cdf[v[-1] + 1] - G[-1]) if len(v) else cdf[-1]


def nonpositive(cdf, v, G, u):
    """The id holding the u-th unit of non-positive weight (u < Q - M), for each u: g = #{j : G_j <= u}, then the CDF
    search for u + PW_g, PW_g = cdf[v_{g-1} + 1] - G_{g-1} the weight of the first g positives."""
    cdf, v, G = np.asarray(cdf, dtype=np.uint64), np.asarray(v, dtype=np.int64), np.asarray(G, dtype=np.uint64)
    u = np.asarray(u, dtype=np.uint64)
    g = np.searchsorted(G, u, side="right")
    j = np.maximum(g - 1, 0)
    pw = np.where(g > 0, cdf[v[j] + 1] - G[j], np.uint64(0)) if len(v) else np.zeros_like(u)
    return search(cdf, u + pw)


def sample_frequency(n, K, cdf, seed, offset):
    """[n, K] int64: b200kge_sample_frequency."""
    cdf = np.asarray(cdf, dtype=np.uint64)
    e = np.arange(n * K, dtype=np.uint64)
    t = nfo.umulhi(nfo.words(e, seed, offset), cdf[-1])
    return search(cdf, t).astype(np.int64).reshape(n, K)


def sample_frequency_filtered(n, K, cdf, seed, offset, triples, slot, keys, offsets, values, below,
                              return_replaced=False):
    """[n, K] int64: b200kge_sample_frequency_filtered (index arrays as filter_csr returns them, below as below_of).
    With return_replaced also the [n, K] bool mask of positions whose first draw was a positive."""
    cdf = np.asarray(cdf, dtype=np.uint64)
    values, offsets = np.asarray(values, dtype=np.int64), np.asarray(offsets, dtype=np.int64)
    below = np.asarray(below, dtype=np.uint64)
    x = sample_frequency(n, K, cdf, seed, offset)
    begin, m, _ = nfo.lookup(keys, offsets, triples[:n], slot)
    out = x.copy()
    replaced = np.zeros((n, K), dtype=bool)
    for i in np.nonzero(m > 0)[0]:
        v, G = values[begin[i]:begin[i] + m[i]], below[begin[i]:begin[i] + m[i]]
        rest = rest_of(cdf, v, G)
        if rest == 0:
            out[i] = -1
            replaced[i] = True
            continue
        hit = np.isin(x[i], v)
        if not hit.any():
            continue
        ks = np.nonzero(hit)[0]
        e = (i * K + ks).astype(np.uint64)
        u = nfo.umulhi(nfo.words(e, seed, offset, nfo.FILTER_DOMAIN), rest)
        out[i, ks] = nonpositive(cdf, v, G, u)
        replaced[i, ks] = True
    return (out, replaced) if return_replaced else out


def _word(e, seed, offset, domain=0):
    block = (e // 2) | domain
    c = philox_ref.philox4x32_10([block & 0xFFFFFFFF, block >> 32, offset & 0xFFFFFFFF, offset >> 32],
                                 (seed & 0xFFFFFFFF, seed >> 32))
    return (c[1] << 32 | c[0]) if e % 2 == 0 else (c[3] << 32 | c[2])


def plain(n, K, q, seed, offset, triples=None, slot=None, positives=None):
    """The definition on Python integers, element by element: the first draw over the prefix of q and, for a positive,
    a walk over the non-positive ids to the one holding the u-th unit of their weight.  positives = {key: set}."""
    cdf = [0]
    for w in q:
        cdf.append(cdf[-1] + int(w))
    Q = cdf[-1]
    out = []
    for i in range(n):
        P = set()
        if positives is not None:
            a, b = nfo.KEY_COLS[slot]
            P = positives.get((int(triples[i][a]), int(triples[i][b])), set())
        rest = Q - sum(int(q[v]) for v in P)
        row = []
        for k in range(K):
            e = i * K + k
            if rest == 0:
                row.append(-1)
                continue
            x = bisect.bisect_right(cdf, (_word(e, seed, offset) * Q) >> 64) - 1
            if x in P:
                u = (_word(e, seed, offset, 1 << 63) * rest) >> 64
                for y in range(len(q)):
                    if y in P:
                        continue
                    if u < q[y]:
                        x = y
                        break
                    u -= q[y]
            row.append(x)
        out.append(row)
    return np.array(out, dtype=np.int64).reshape(n, K)
