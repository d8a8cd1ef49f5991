"""TEST INFRASTRUCTURE: b200kge_sample_uniform_filtered (kge_b200/csrc/rowwise.cu) restated on numpy, vectorised over
all elements of a call, and the definition it implements, by brute force.

Element e = i*K + k takes word pair (e & 1) of Philox block (e // 2, offset) under key seed and maps it to
x = floor(r * V / 2^64) (b200kge_sample_uniform's draw).  If x is a positive of row i's key, the output is the u-th
non-positive id, u = floor(r' * (V - m) / 2^64), r' the same word pair of block (e // 2 | 2^63, offset) under the same
key; m is the key's number of distinct positives.  Absent keys are unfiltered; rows with m >= V get -1."""
from __future__ import annotations

import numpy as np

from philox_np import philox4x32_10

M32 = np.uint64(0xFFFFFFFF)
S32 = np.uint64(32)
FILTER_DOMAIN = 1 << 63
KEY_COLS = {0: (1, 2), 1: (0, 2), 2: (0, 1)}       # (p, o) for S, (s, o) for P, (s, p) for O


def umulhi(a, b):
    """floor(a * b / 2^64) for uint64 arrays, from 32-bit limbs."""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    a_lo, a_hi, b_lo, b_hi = a & M32, a >> S32, b & M32, b >> S32
    p0, p1, p2, p3 = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (p0 >> S32) + (p1 & M32) + (p2 & M32)
    return p3 + (p1 >> S32) + (p2 >> S32) + (mid >> S32)


def words(e, seed, offset, domain=0):
    """The 64-bit word of element(s) e: pair (e & 1) of block (e // 2 | domain, offset) under key seed."""
    e = np.asarray(e, dtype=np.uint64)
    block = (e >> np.uint64(1)) | np.uint64(domain)
    c = philox4x32_10(block & M32, block >> S32, offset & 0xFFFFFFFF, (offset >> 32) & 0xFFFFFFFF,
                      (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    odd = (e & np.uint64(1)).astype(bool)
    return np.where(odd, (c[3] << S32) | c[2], (c[1] << S32) | c[0])


def sample_uniform(n, K, vocab, seed, offset):
    """[n, K] int64: b200kge_sample_uniform."""
    e = np.arange(n * K, dtype=np.uint64)
    return umulhi(words(e, seed, offset), vocab).astype(np.int64).reshape(n, K)


def row_keys(triples, slot):
    a, b = KEY_COLS[slot]
    t = np.asarray(triples, dtype=np.int64)
    return t[:, a], t[:, b]


def lookup(keys, offsets, triples, slot):
    """(begin, m) per row of triples: the key's slice of the index's values (m = 0 for an absent key)."""
    keys, offsets = np.asarray(keys, dtype=np.int64).reshape(-1, 2), np.asarray(offsets, dtype=np.int64)
    a, b = row_keys(triples, slot)
    if len(keys) == 0:
        zero = np.zeros(len(a), dtype=np.int64)
        return zero, zero, zero - 1
    comp = keys[:, 0] * (1 << 31) + keys[:, 1]
    q = a * (1 << 31) + b
    j = np.minimum(np.searchsorted(comp, q), len(comp) - 1)
    hit = comp[j] == q
    begin = np.where(hit, offsets[j], 0)
    m = np.where(hit, offsets[j + 1] - offsets[j], 0)
    return begin, m, np.where(hit, j, -1)


def sample_uniform_filtered(n, K, vocab, seed, offset, triples, slot, keys, offsets, values, return_replaced=False):
    """[n, K] int64: b200kge_sample_uniform_filtered (index arrays as filter_csr returns them).  With return_replaced
    also the [n, K] bool mask of positions whose first draw was a positive."""
    values, offsets = np.asarray(values, dtype=np.int64), np.asarray(offsets, dtype=np.int64)
    V = int(vocab)
    x = sample_uniform(n, K, V, seed, offset)
    begin, m, kidx = lookup(keys, offsets, triples[:n], slot)
    out = x.copy()
    replaced = np.zeros((n, K), dtype=bool)
    rows = np.nonzero(m > 0)[0]
    if len(rows):
        # every key's values sit in one sorted run: key j's run sorts before key j+1's in (key index, value) order
        nk = len(offsets) - 1
        owner = np.repeat(np.arange(nk), offsets[1:] - offsets[:-1])
        comp = owner * V + values
        local = np.arange(len(values)) - offsets[owner]
        comp2 = owner * (V + 1) + (values - local)
        xr = x[rows]
        q = kidx[rows][:, None] * V + xr
        pos = np.searchsorted(comp, q)
        hit = (pos < len(comp)) & (comp[np.minimum(pos, len(comp) - 1)] == q)
        hit &= (m[rows] < V)[:, None]
        ri, ki = np.nonzero(hit)
        i = rows[ri]
        e = (i * K + ki).astype(np.uint64)
        mm = m[i]
        u = umulhi(words(e, seed, offset, FILTER_DOMAIN), (V - mm).astype(np.uint64)).astype(np.int64)
        c = np.searchsorted(comp2, kidx[i] * (V + 1) + u, side="right") - offsets[kidx[i]]
        out[i, ki] = u + c
        replaced[i, ki] = True
    out[m >= V] = -1
    replaced[m >= V] = True                          # every id is a positive there
    return (out, replaced) if return_replaced else out


def brute_force(n, K, vocab, seed, offset, triples, slot, positives):
    """The definition, element by element: positives = {key: set of ids}; the u-th id of sorted(range(V) - P)."""
    x = sample_uniform(n, K, vocab, seed, offset)
    a, b = row_keys(triples, slot)
    out = np.empty((n, K), dtype=np.int64)
    for i in range(n):
        P = positives.get((int(a[i]), int(b[i])), set())
        if len(P) >= vocab:
            out[i] = -1
            continue
        nonpos = None
        for k in range(K):
            if int(x[i, k]) not in P:
                out[i, k] = x[i, k]
                continue
            if nonpos is None:
                nonpos = sorted(set(range(vocab)) - P)
            e = i * K + k
            u = int(umulhi(words(e, seed, offset, FILTER_DOMAIN), vocab - len(P)))
            out[i, k] = nonpos[u]
    return out


def positives_of(split, slot):
    """{key: set of values} of a split [N, 3] for a slot: the dict-of-sets definition of the filtering index."""
    a, b = KEY_COLS[slot]
    d = {}
    for t in np.asarray(split, dtype=np.int64).tolist():
        d.setdefault((t[a], t[b]), set()).add(t[slot])
    return d
