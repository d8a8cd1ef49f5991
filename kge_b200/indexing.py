"""Host-side mirror of LibKGE's KvsAllIndex (kge/indexing.py:10-194) on the native library.

Same attributes (`_keys`, `_values_offset`, `_values`) and accessors (`__getitem__`, `get`, `get_all`,
`__len__`, `keys`, `values`, `items`) as the reference class, so `TrainingJobKvsAll` and
`EntityRankingJob` can use it unchanged; the sort / unique / lookup loops run in C++
(`b200kge_kvsall_*`, kge_b200/csrc/hostindex.cu) instead of numpy + a numba dict.  In addition the CSR
forms (`get_all_csr`, `collate_csr`) are what the device label / filter epilogues take instead of a
densified coordinate tensor.  CPU only: nothing here touches the GPU.
"""
from __future__ import annotations

from typing import Iterator, List, Optional, Tuple

import torch

from . import _lib

S, P, O = 0, 1, 2
_KEY_COLS = {"sp": ([S, P], O), "po": ([P, O], S), "so": ([S, O], P)}


def _i64(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(device="cpu", dtype=torch.int64).contiguous()


class KvsAllIndex:
    def __init__(self, triples: torch.Tensor, key_cols: List[int], value_col: int, default_factory: type = list):
        self.key_cols = list(key_cols)
        self.value_col = int(value_col)
        self.default_factory = default_factory
        self.default_index_of_key = -1
        self._dtype = triples.dtype
        tri = _i64(triples).view(-1, 3)
        n = tri.shape[0]
        keys = torch.empty((n, 2), dtype=torch.int64)
        offs = torch.empty((n + 1,), dtype=torch.int64)
        vals = torch.empty((n,), dtype=torch.int64)
        import ctypes as C

        nk = C.c_int64(0)
        _lib.check(_lib.load().b200kge_kvsall_index_build(
            tri.data_ptr(), n, self.key_cols[0], self.key_cols[1], self.value_col,
            keys.data_ptr(), offs.data_ptr(), vals.data_ptr(), C.byref(nk)))
        k = nk.value
        self._keys64 = keys[:k].clone()
        self._offsets64 = offs[: k + 1].clone()
        self._values64 = vals
        # the reference keeps keys / values in the triples' dtype and the offsets as int32
        self._keys = self._keys64.to(self._dtype)
        self._values_offset = self._offsets64.int()
        self._values = self._values64.to(self._dtype)

    # -- reference accessors ---------------------------------------------------------------------------
    def __len__(self) -> int:
        return self._keys64.shape[0]

    def _index_of(self, key) -> int:
        k = (int(key[0]), int(key[1]))
        lo, hi = 0, len(self)
        while lo < hi:
            mid = (lo + hi) // 2
            if (int(self._keys64[mid, 0]), int(self._keys64[mid, 1])) < k:
                lo = mid + 1
            else:
                hi = mid
        if lo < len(self) and (int(self._keys64[lo, 0]), int(self._keys64[lo, 1])) == k:
            return lo
        return -1

    def __getitem__(self, key, default_return_value=None) -> torch.Tensor:
        i = self._index_of(key)
        if i < 0:
            return self.default_factory() if default_return_value is None else default_return_value
        return self._values[int(self._offsets64[i]): int(self._offsets64[i + 1])]

    def get(self, key, default_return_value=None) -> torch.Tensor:
        return self.__getitem__(key, default_return_value)

    def get_all_csr(self, keys: torch.Tensor, col_shift: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """(offsets [n+1], cols [nnz]) int64: values of every query key, absent keys empty."""
        q = _i64(keys).view(-1, 2)
        n = q.shape[0]
        offs = torch.empty((n + 1,), dtype=torch.int64)
        lib = _lib.load()
        args = (self._keys64.data_ptr(), self._offsets64.data_ptr(), self._values64.data_ptr(), len(self),
                q.data_ptr(), n, int(col_shift), offs.data_ptr())
        _lib.check(lib.b200kge_kvsall_lookup(*args, None))
        cols = torch.empty((int(offs[n]),), dtype=torch.int64)
        _lib.check(lib.b200kge_kvsall_lookup(*args, cols.data_ptr()))
        return offs, cols

    def get_all(self, keys: torch.Tensor) -> torch.Tensor:
        """[m,2] int32: (position of the key in `keys`, value) for all values of all keys (indexing.py:155-166)."""
        offs, cols = self.get_all_csr(keys)
        rows = torch.repeat_interleave(torch.arange(offs.numel() - 1), offs[1:] - offs[:-1])
        return torch.stack([rows, cols], 1).int()

    def collate_csr(self, examples: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(queries [b,2], offsets [b+1], cols [nnz]) for a batch of example (= key) indexes: the collate
        function of KvsAll training for one query type (train_KvsAll.py:116-203) with CSR labels."""
        ex = _i64(examples).view(-1)
        b = ex.numel()
        queries = torch.empty((b, 2), dtype=torch.int64)
        offs = torch.empty((b + 1,), dtype=torch.int64)
        lib = _lib.load()
        args = (self._keys64.data_ptr(), self._offsets64.data_ptr(), self._values64.data_ptr(), len(self),
                ex.data_ptr(), b, queries.data_ptr(), offs.data_ptr())
        _lib.check(lib.b200kge_kvsall_gather(*args, None))
        cols = torch.empty((int(offs[b]),), dtype=torch.int64)
        _lib.check(lib.b200kge_kvsall_gather(*args, cols.data_ptr()))
        return queries, offs, cols

    def keys(self) -> Iterator[Tuple[int, int]]:
        return iter([(int(a), int(b)) for a, b in self._keys64.tolist()])

    def values(self) -> List[torch.Tensor]:
        return [self._values[int(self._offsets64[i]): int(self._offsets64[i + 1])] for i in range(len(self))]

    def items(self):
        return zip(self.keys(), self.values())


def index_KvsAll(triples: torch.Tensor, key: str) -> KvsAllIndex:
    """Index from `key` ("sp" | "po" | "so") to the remaining slot (indexing.py:197-228)."""
    if key not in _KEY_COLS:
        raise ValueError(f"unknown key {key!r}: expected one of sp, po, so")
    cols, val = _KEY_COLS[key]
    return KvsAllIndex(triples, cols, val, list)


def filter_csr(index, vocab: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, int]:
    """(keys [k,2], offsets [k+1], values [nnz], largest count) int64: the filter index of negative sampling
    (b200kge_filter_index_build) from a KvsAllIndex — the reference's or this module's, both have `_keys`,
    `_values_offset` and `_values`.  Keys sorted and unique, values sorted and distinct per key, all in [0, vocab)."""
    keys, offs, vals = _i64(index._keys).view(-1, 2), _i64(index._values_offset).view(-1), _i64(index._values).view(-1)
    k = keys.shape[0]
    cap = max(int(offs[k] - offs[0]), 0)
    keys_out = torch.empty((k, 2), dtype=torch.int64)
    offs_out = torch.empty((k + 1,), dtype=torch.int64)
    vals_out = torch.empty((cap,), dtype=torch.int64)
    import ctypes as C

    nk, mx = C.c_int64(0), C.c_int64(0)
    _lib.check(_lib.load().b200kge_filter_index_build(
        keys.data_ptr(), offs.data_ptr(), vals.data_ptr(), k, int(vocab), keys_out.data_ptr(), offs_out.data_ptr(),
        vals_out.data_ptr(), C.byref(nk), C.byref(mx)))
    nk = nk.value
    return keys_out[:nk].clone(), offs_out[: nk + 1].clone(), vals_out[: int(offs_out[nk])].clone(), mx.value


def frequency_cdf(counts: torch.Tensor, smoothing: float) -> torch.Tensor:
    """cdf [V+1] int64 (every entry <= 2^62): the exclusive prefix of the integer weights of frequency sampling,
    q_x = round((counts[x] + smoothing) * 2^s) with the largest s that keeps their sum within 2^62
    (b200kge_frequency_cdf_build).  ValueError for a negative count, a negative or non-finite smoothing, or all-zero
    weights."""
    c = _i64(counts).view(-1)
    cdf = torch.empty((c.numel() + 1,), dtype=torch.int64)
    _lib.check(_lib.load().b200kge_frequency_cdf_build(c.data_ptr(), c.numel(), float(smoothing), cdf.data_ptr()))
    return cdf


def frequency_below(cdf: torch.Tensor, offsets: torch.Tensor, values: torch.Tensor) -> Tuple[torch.Tensor, int, int]:
    """(below [nnz] int64, number of keys, first key index or -1): for every value v_j of a key of a filter index
    (filter_csr's offsets / values), the weight of the key's non-positives below v_j under `cdf`, and the keys whose
    positives carry all the weight (b200kge_frequency_filter_build)."""
    cdf, offs, vals = _i64(cdf).view(-1), _i64(offsets).view(-1), _i64(values).view(-1)
    below = torch.empty_like(vals)
    import ctypes as C

    full, first = C.c_int64(0), C.c_int64(0)
    _lib.check(_lib.load().b200kge_frequency_filter_build(
        cdf.data_ptr(), cdf.numel() - 1, offs.data_ptr(), vals.data_ptr(), offs.numel() - 1, below.data_ptr(),
        C.byref(full), C.byref(first)))
    return below, full.value, first.value


def sp_po_label_csr(triples: torch.Tensor, num_entities: int, sp_index: KvsAllIndex, po_index: KvsAllIndex,
                    ) -> Tuple[torch.Tensor, torch.Tensor]:
    """CSR over the [n, 2E] label / filter matrix of a batch of (s,p,o) triples: known objects of (s,p,?) in
    columns [0,E), known subjects of (?,p,o) in columns [E,2E)  (get_sp_po_coords_from_spo_batch,
    kge/job/util.py:6-30; the reference concatenates all sp coordinates, then all po coordinates — here they
    are merged per row, which is the same set of coordinates)."""
    tri = _i64(triples).view(-1, 3)
    o_sp, c_sp = sp_index.get_all_csr(tri[:, [S, P]])
    o_po, c_po = po_index.get_all_csr(tri[:, [P, O]], col_shift=num_entities)
    n = tri.shape[0]
    cnt = (o_sp[1:] - o_sp[:-1]) + (o_po[1:] - o_po[:-1])
    offs = torch.zeros((n + 1,), dtype=torch.int64)
    offs[1:] = torch.cumsum(cnt, 0)
    cols = torch.empty((int(offs[n]),), dtype=torch.int64)
    # per-row merge: [sp values | po values]
    sp_len = o_sp[1:] - o_sp[:-1]
    row_sp = torch.repeat_interleave(torch.arange(n), sp_len)
    pos_sp = offs[:-1][row_sp] + (torch.arange(c_sp.numel()) - o_sp[:-1][row_sp])
    cols[pos_sp] = c_sp
    po_len = o_po[1:] - o_po[:-1]
    row_po = torch.repeat_interleave(torch.arange(n), po_len)
    pos_po = offs[:-1][row_po] + sp_len[row_po] + (torch.arange(c_po.numel()) - o_po[:-1][row_po])
    cols[pos_po] = c_po
    return offs, cols


def csr_to_coords(offsets: torch.Tensor, cols: torch.Tensor) -> torch.Tensor:
    """[nnz,2] (row, col) coordinates of a CSR pattern — the layout coord_to_sparse_tensor consumes."""
    rows = torch.repeat_interleave(torch.arange(offsets.numel() - 1), offsets[1:] - offsets[:-1])
    return torch.stack([rows, cols], 1)
