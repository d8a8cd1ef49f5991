"""Tensor-level façade over the C ABI: torch CUDA tensors in, torch CUDA tensors out.

torch is used for device memory (caching allocator), streams and nothing else: every number is
produced by libb200kge's hand-written sm_90a kernels.  All functions raise on CPU tensors.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch

from . import _lib
from ._lib import LOSS, MODELS, NS_IMPL, PREC, Dropout, Labels, Rows, SP_, _PO

S, P, O = 0, 1, 2


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "kge_b200 runs on CUDA (sm_90) tensors only; there is no CPU path "
                f"(got a tensor on {t.device})"
            )


def _f32(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise TypeError(f"expected float32 embeddings, got {t.dtype}")
    if t.dim() != 2:
        raise ValueError(f"expected a 2-D embedding matrix, got shape {tuple(t.shape)}")
    if t.stride(1) != 1:
        t = t.contiguous()
    return t


def _i64(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if t.dim() != 1:
        t = t.reshape(-1)
    if t.dtype != torch.int64 or not t.is_contiguous():
        t = t.long().contiguous()  # lookup_embedder.py:97 does indexes.long()
    return t


def _f32_rows(t: torch.Tensor) -> torch.Tensor:
    """t as float32 with unit column stride (a row stride the kernels can take), copied only if it is not already."""
    return t if (t.dtype == torch.float32 and t.stride(1) == 1) else t.float().contiguous()


def _i64_block(t: torch.Tensor) -> torch.Tensor:
    """t (triples [n, 3], negatives [n, K]) as a contiguous int64 block, copied only if it is not already."""
    return t if (t.dtype == torch.int64 and t.is_contiguous()) else t.long().contiguous()


class _Keep:
    """Keeps tensors alive for the duration of a call (the C side borrows raw pointers)."""

    def __init__(self):
        self.refs = []

    def rows(self, base: torch.Tensor, idx: Optional[torch.Tensor] = None) -> Rows:
        base = _f32(base)
        idx = _i64(idx)
        self.refs += [base, idx]
        r = Rows()
        r.base = base.data_ptr()
        r.idx = idx.data_ptr() if idx is not None else None
        r.rows = idx.numel() if idx is not None else base.shape[0]
        r.ld = base.stride(0) if base.shape[0] > 1 else max(base.shape[1], base.stride(0))
        r.dim = base.shape[1]
        return r


def _stream(dev) -> C.c_void_p:
    """The operands' current stream.  The library launches on the CURRENT device, so follow the operands when they live
    elsewhere (`job.device: cuda:1` in a process that never called set_device, e.g. LibKGE's search workers,
    kge/job/search.py:36-40); a no-op when the devices already agree."""
    idx = dev.index if isinstance(dev, torch.device) else torch.device(dev).index
    if idx is not None and idx != torch.cuda.current_device():
        torch.cuda.set_device(idx)
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _workspace(model_id: int, n: int, m: int, D: int, has_idx: bool, dev) -> torch.Tensor:
    nbytes = _lib.load().b200kge_workspace_bytes(model_id, n, m, D, 1 if has_idx else 0)
    # torch's caching allocator raises torch.cuda.OutOfMemoryError ("CUDA out of memory") on failure
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


class DropoutKey(NamedTuple):
    """Embedding dropout of one training sub-batch (b200kge_dropout_t): the rates of the entity and relation embedders
    and the mask key.  Every mask element is a pure function of (seed, call, stream, global row, column), so the
    backward, given the same key, regenerates the forward's masks."""
    p_ent: float
    p_rel: float
    seed: int
    call: int
    row_base: int = 0

    def struct(self) -> Dropout:
        return Dropout(float(self.p_ent), float(self.p_rel), int(self.seed) & (2 ** 64 - 1),
                       int(self.call) & (2 ** 64 - 1), int(self.row_base))


def dropout_mask(p: float, seed: int, call: int, stream: int, rows: int, dim: int, row_base: int = 0,
                 device="cuda") -> torch.Tensor:
    """The keep mask [rows, dim] (uint8) of draw `stream` (0-5 and 24-26, include/b200kge.h) over global rows
    [row_base, row_base + rows)."""
    out = torch.empty((rows, dim), dtype=torch.uint8, device=device)
    _require_cuda(out)
    _lib.check(_lib.load().b200kge_dropout_mask(float(p), int(seed) & (2 ** 64 - 1), int(call) & (2 ** 64 - 1),
                                                int(stream), int(row_base), rows, dim, out.data_ptr(),
                                                _stream(out.device)))
    return out


def device_ok() -> bool:
    return _lib.load().b200kge_device_ok() == 0


def launch_count(reset: bool = False) -> int:
    return int(_lib.load().b200kge_launch_count(1 if reset else 0))


def profile_enable(on: bool = True) -> None:
    _lib.load().b200kge_profile_enable(1 if on else 0)


def profile_last_ms() -> float:
    ms = C.c_float(0.0)
    _lib.check(_lib.load().b200kge_profile_last_ms(C.byref(ms)))
    return float(ms.value)


# ------------------------------------------------------------------------------------------------
def score_spo(model: str, ent_s, rel, ent_o, s=None, p=None, o=None, l_norm: float = 1.0):
    """Row-wise scores.  With indexes: tables + gather fused (KgeModel.score_spo); without:
    already-gathered embeddings (RelationalScorer.score_emb(..., "spo"))."""
    _require_cuda(ent_s, rel, ent_o)
    lib, k = _lib.load(), _Keep()
    rs, rp, ro = k.rows(ent_s, s), k.rows(rel, p), k.rows(ent_o, o)
    n = int(rs.rows)
    if rp.rows != n or ro.rows != n:
        raise ValueError("spo scoring needs the same number of s, p and o rows")
    out = torch.empty(n, dtype=torch.float32, device=ent_s.device)
    _lib.check(lib.b200kge_score_spo(MODELS[model], l_norm, C.byref(rs), C.byref(rp), C.byref(ro), n,
                                     out.data_ptr(), _stream(ent_s.device)))
    return out


def score_1vsN(model: str, combine: str, q_tab, rel, cand_tab, q=None, p=None, cand=None,
               l_norm: float = 1.0, precision: str = "auto", out: Optional[torch.Tensor] = None):
    """[n, m] scores of n (entity, relation) rows against m candidate entities.

    combine "sp_": q rows are subjects, candidates are objects; "_po": q rows are objects,
    candidates are subjects (kge_model.py:164-181)."""
    if combine not in ("sp_", "_po"):
        raise ValueError('cannot handle combine="{}"'.format(combine))
    _require_cuda(q_tab, rel, cand_tab)
    lib, k = _lib.load(), _Keep()
    rq, rp, rc = k.rows(q_tab, q), k.rows(rel, p), k.rows(cand_tab, cand)
    n, m = int(rq.rows), int(rc.rows)
    if rp.rows != n:
        raise ValueError("need as many relation rows as entity rows")
    dev = q_tab.device
    if out is None:
        out = torch.empty((n, m), dtype=torch.float32, device=dev)
    ws = _workspace(MODELS[model], n, m, rq.dim, cand is not None, dev)
    _lib.check(lib.b200kge_score_1vsN(MODELS[model], SP_ if combine == "sp_" else _PO, l_norm,
                                      PREC[precision], C.byref(rq), C.byref(rp), C.byref(rc), n,
                                      out.data_ptr(), out.stride(0), ws.data_ptr(), ws.numel(),
                                      _stream(dev)))
    return out


def score_sp_po(model: str, ent, rel, s, p, o, entity_subset=None, l_norm: float = 1.0,
                precision: str = "auto", out: Optional[torch.Tensor] = None, ent_o=None, cand_tab=None):
    """[n, 2m] = [score_sp | score_po] in one launch sequence (kge_model.py:749-789).

    Index level: ent / rel are the tables, s / p / o index vectors.  Embedding level (s = p = o = None): ent, rel,
    ent_o are already-gathered [n, .] subject / relation / object rows and cand_tab the candidate table.
    `out` (optional) is a caller-owned [n, >= 2m] float32 block with unit column stride (e.g. a slice of an
    all-gather buffer): the two halves are written at columns [0, m) and [m, 2m)."""
    _require_cuda(ent, rel)
    lib, k = _lib.load(), _Keep()
    rs, rp, ro = k.rows(ent, s), k.rows(rel, p), k.rows(ent if ent_o is None else ent_o, o)
    rc = k.rows(ent if cand_tab is None else cand_tab, entity_subset)
    n, m = int(rs.rows), int(rc.rows)
    dev = ent.device
    if out is None:
        out = torch.empty((n, 2 * m), dtype=torch.float32, device=dev)
    elif out.dtype != torch.float32 or out.stride(1) != 1 or out.shape[0] < n or out.shape[1] < 2 * m:
        raise ValueError("out must be a float32 [n, >= 2m] block with unit column stride")
    ws = _workspace(MODELS[model], n, m, rs.dim, entity_subset is not None, dev)
    _lib.check(lib.b200kge_score_sp_po(MODELS[model], l_norm, PREC[precision], C.byref(rs), C.byref(rp),
                                       C.byref(ro), C.byref(rc), n, out.data_ptr(), out.stride(0),
                                       ws.data_ptr(), ws.numel(), _stream(dev)))
    return out


def score_sp_po_bcast(model: str, s_emb, rel, p, o_emb, cand_tab, out_ptr: int, peer_ptrs, ldo: int, col_block: int,
                      l_norm: float = 1.0, precision: str = "auto"):
    """score_sp_po whose epilogue stores go to this rank's buffer (raw device address out_ptr, already offset to the
    shard's first column) AND to the peer-mapped buffers `peer_ptrs` of the other ranks at the same offsets — the
    all-gather of per-shard logits fused into the scoring kernel (include/b200kge.h: b200kge_score_sp_po_bcast)."""
    _require_cuda(s_emb, rel, o_emb, cand_tab)
    lib, k = _lib.load(), _Keep()
    rs, rp, ro, rc = k.rows(s_emb), k.rows(rel, p), k.rows(o_emb), k.rows(cand_tab)
    n, m = int(rs.rows), int(rc.rows)
    dev = s_emb.device
    arr = (C.c_void_p * max(1, len(peer_ptrs)))(*[C.c_void_p(int(x)) for x in peer_ptrs])
    ws = _workspace(MODELS[model], n, m, rs.dim, False, dev)
    _lib.check(lib.b200kge_score_sp_po_bcast(MODELS[model], l_norm, PREC[precision], C.byref(rs), C.byref(rp),
                                             C.byref(ro), C.byref(rc), n, C.c_void_p(int(out_ptr)), arr,
                                             len(peer_ptrs), ldo, col_block, ws.data_ptr(), ws.numel(), _stream(dev)))


def rank_sp_po(model: str, s_tab, rel, o_tab, cand_tab, true_scores, s=None, p=None, o=None, cand=None,
               filter_labels=None, rtol: float = 1e-4, atol: float = 1e-5, l_norm: float = 1.0,
               precision: str = "auto", rank=None, ties=None):
    """Both directions of one batch's ranking against one chunk of candidates in ONE launch sequence: rows
    0..n-1 = sp_ queries, n..2n-1 = _po queries; true_scores / rank / ties are [2n] in that order (rank / ties
    int64, accumulated into); filter_labels (optional) [2n, m]."""
    _require_cuda(s_tab, rel, o_tab, cand_tab, true_scores, filter_labels)
    lib, k = _lib.load(), _Keep()
    rs, rp, ro, rc = k.rows(s_tab, s), k.rows(rel, p), k.rows(o_tab, o), k.rows(cand_tab, cand)
    n, m = int(rs.rows), int(rc.rows)
    dev = s_tab.device
    t = true_scores.reshape(-1).float().contiguous()
    if t.numel() != 2 * n:
        raise ValueError("true_scores must hold 2n values: sp_ rows first, then _po rows")
    if rank is None:
        rank = torch.zeros(2 * n, dtype=torch.int64, device=dev)
    if ties is None:
        ties = torch.zeros(2 * n, dtype=torch.int64, device=dev)
    f = None
    if filter_labels is not None:
        f = _f32_rows(filter_labels)
    ws = _workspace(MODELS[model], n, m, rs.dim, cand is not None, dev)
    _lib.check(lib.b200kge_rank_sp_po(
        MODELS[model], l_norm, PREC[precision], C.byref(rs), C.byref(rp), C.byref(ro), C.byref(rc), n, t.data_ptr(),
        f.data_ptr() if f is not None else None, f.stride(0) if f is not None else 0, rtol, atol, rank.data_ptr(),
        ties.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)))
    return rank, ties


def rank_sp_po_csr(model: str, s_tab, rel, o_tab, cand_tab, true_scores, filter_off, filter_col, own_col=None,
                   s=None, p=None, o=None, rtol: float = 1e-4, atol: float = 1e-5, l_norm: float = 1.0,
                   precision: str = "auto", rank=None, ties=None):
    """rank_sp_po with the known-answer filter as CSR over the stacked rows (sp_ rows, then _po rows): row r lists
    sorted candidate columns filter_col[filter_off[r]:filter_off[r+1]]; own_col[r] (the row's own answer) stays in.
    Raises NotImplementedError when the shape / model is not served by the pre-split tensor-core kernel."""
    _require_cuda(s_tab, rel, o_tab, cand_tab, true_scores, filter_off, filter_col, own_col)
    lib, k = _lib.load(), _Keep()
    rs, rp, ro, rc = k.rows(s_tab, s), k.rows(rel, p), k.rows(o_tab, o), k.rows(cand_tab)
    n, m = int(rs.rows), int(rc.rows)
    dev = s_tab.device
    t = true_scores.reshape(-1).float().contiguous()
    offs, cols = _i64(filter_off), _i64(filter_col)
    own = _i64(own_col)
    if t.numel() != 2 * n or offs.numel() != 2 * n + 1:
        raise ValueError("true_scores / filter_off must cover the 2n stacked rows")
    if rank is None:
        rank = torch.zeros(2 * n, dtype=torch.int64, device=dev)
    if ties is None:
        ties = torch.zeros(2 * n, dtype=torch.int64, device=dev)
    ws = _workspace(MODELS[model], n, m, rs.dim, False, dev)
    _lib.check(lib.b200kge_rank_sp_po_csr(
        MODELS[model], l_norm, PREC[precision], C.byref(rs), C.byref(rp), C.byref(ro), C.byref(rc), n, t.data_ptr(),
        offs.data_ptr(), cols.data_ptr() if cols.numel() else None, own.data_ptr() if own is not None else None,
        rtol, atol, rank.data_ptr(), ties.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)))
    return rank, ties


def rank_sp_po_eval(model: str, ent, rel, s, p, o, true_scores, own_col, filter_off, filter_col, test_off=None,
                    test_col=None, rtol: float = 1e-4, atol: float = 1e-5, l_norm: float = 1.0, precision: str = "auto",
                    num_relations: int = 0):
    """Every ranking of one evaluation batch from ONE scoring pass over the whole table (b200kge_rank_sp_po_eval).

    Stacked rows: 0..n-1 the sp_ queries (s, p), n..2n-1 the _po queries (p, o), or with num_relations = R > 0 the sp_
    queries (o, p + R) of a reciprocal-relations base model.  true_scores / own_col are [2n]; (filter_off, filter_col)
    the CSR of the known answers and (test_off, test_col) (optional) that of the test answers not among them, both
    sorted and unique per row.  Returns (rank, ties, own_score): rank / ties int64 [2 or 3, 2n] (raw, _filt[,
    _filt_test]), own_score [2n] the scores the kernel computed at own_col."""
    _require_cuda(ent, rel, s, p, o, true_scores, own_col, filter_off, filter_col, test_off, test_col)
    if (test_off is None) != (test_col is None):
        raise ValueError("test_off and test_col go together")
    lib, k = _lib.load(), _Keep()
    re, rr = k.rows(ent), k.rows(rel)
    si, pi, oi = _i64(s), _i64(p), _i64(o)
    n = si.numel()
    if pi.numel() != n or oi.numel() != n:
        raise ValueError("s, p and o must have the same length")
    dev = ent.device
    t = true_scores.reshape(-1).float().contiguous()
    own = _i64(own_col)
    offs, cols = _i64(filter_off), _i64(filter_col)
    toffs, tcols = _i64(test_off), _i64(test_col)
    if t.numel() != 2 * n or own.numel() != 2 * n or offs.numel() != 2 * n + 1 or (
            toffs is not None and toffs.numel() != 2 * n + 1):
        raise ValueError("true_scores / own_col / the CSR offsets must cover the 2n stacked rows")
    k.refs += [si, pi, oi, t, own, offs, cols, toffs, tcols]
    nr = 2 if toffs is None else 3
    rank = torch.zeros((nr, 2 * n), dtype=torch.int64, device=dev)
    ties = torch.zeros((nr, 2 * n), dtype=torch.int64, device=dev)
    own_score = torch.empty(2 * n, dtype=torch.float32, device=dev)
    ws = _workspace(MODELS[model], n, re.rows, re.dim, False, dev)

    def ptr(x):
        return x.data_ptr() if x is not None and x.numel() else None
    _lib.check(lib.b200kge_rank_sp_po_eval(
        MODELS[model], l_norm, PREC[precision], C.byref(re), C.byref(rr), int(num_relations), si.data_ptr(),
        pi.data_ptr(), oi.data_ptr(), n, t.data_ptr(), own.data_ptr(), offs.data_ptr(), ptr(cols),
        toffs.data_ptr() if toffs is not None else None, ptr(tcols), rtol, atol, rank.data_ptr(), ties.data_ptr(),
        own_score.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)))
    return rank, ties, own_score


def shard_gather_rows(shard: torch.Tensor, lo: int, idx: torch.Tensor, out: Optional[torch.Tensor] = None):
    """This rank's contribution to the query-row exchange of an entity-sharded table: out[i] = shard[idx[i] - lo]
    if lo <= idx[i] < lo + rows else 0 (one kernel, no host synchronisation)."""
    _require_cuda(shard, idx)
    lib, k = _lib.load(), _Keep()
    rsh = k.rows(shard)
    ix = _i64(idx)
    n = ix.numel()
    if out is None:
        out = torch.empty((n, shard.shape[1]), dtype=torch.float32, device=shard.device)
    _lib.check(lib.b200kge_shard_gather_rows(C.byref(rsh), int(lo), ix.data_ptr(), n, out.data_ptr(), out.stride(0),
                                             _stream(shard.device)))
    return out


def _labels(k: _Keep, labels: torch.Tensor) -> Labels:
    lab = Labels()
    if labels.dim() == 1:
        li = _i64(labels)
        k.refs.append(li)
        lab.idx, lab.dense, lab.ldl = li.data_ptr(), None, 0
    else:
        ld = _f32_rows(labels)
        k.refs.append(ld)
        lab.idx, lab.dense, lab.ldl = None, ld.data_ptr(), ld.stride(0)
    return lab


def score_1vsN_loss(model: str, combine: str, q_tab, rel, cand_tab, labels, q=None, p=None, cand=None,
                    loss: str = "bce", offset: float = 0.0, l_norm: float = 1.0, precision: str = "auto",
                    return_rows: bool = False):
    """Fused scoring + KgeLoss (sum reduction): returns a 0-d tensor (and per-row terms)."""
    _require_cuda(q_tab, rel, cand_tab, labels)
    lib, k = _lib.load(), _Keep()
    rq, rp, rc = k.rows(q_tab, q), k.rows(rel, p), k.rows(cand_tab, cand)
    n, m = int(rq.rows), int(rc.rows)
    dev = q_tab.device
    lab = _labels(k, labels)
    out = torch.empty((), dtype=torch.float32, device=dev)
    rows = torch.empty(n, dtype=torch.float32, device=dev) if return_rows else None
    ws = _workspace(MODELS[model], n, m, rq.dim, cand is not None, dev)
    _lib.check(lib.b200kge_score_1vsN_loss(
        MODELS[model], SP_ if combine == "sp_" else _PO, l_norm, PREC[precision], C.byref(rq), C.byref(rp),
        C.byref(rc), n, C.byref(lab), LOSS[loss], offset, out.data_ptr(),
        rows.data_ptr() if rows is not None else None, ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, rows) if return_rows else out


def score_1vsN_rank(model: str, combine: str, q_tab, rel, cand_tab, true_scores, q=None, p=None, cand=None,
                    filter_labels=None, rtol: float = 1e-4, atol: float = 1e-5, l_norm: float = 1.0,
                    precision: str = "auto", rank=None, ties=None):
    """Fused scoring + rank/tie counting for one chunk of candidates; accumulates into rank/ties."""
    _require_cuda(q_tab, rel, cand_tab, true_scores, filter_labels)
    lib, k = _lib.load(), _Keep()
    rq, rp, rc = k.rows(q_tab, q), k.rows(rel, p), k.rows(cand_tab, cand)
    n, m = int(rq.rows), int(rc.rows)
    dev = q_tab.device
    t = true_scores.reshape(-1).float().contiguous()
    if rank is None:
        rank = torch.zeros(n, dtype=torch.int64, device=dev)
    if ties is None:
        ties = torch.zeros(n, dtype=torch.int64, device=dev)
    f = None
    if filter_labels is not None:
        f = _f32_rows(filter_labels)
    ws = _workspace(MODELS[model], n, m, rq.dim, cand is not None, dev)
    _lib.check(lib.b200kge_score_1vsN_rank(
        MODELS[model], SP_ if combine == "sp_" else _PO, l_norm, PREC[precision], C.byref(rq), C.byref(rp),
        C.byref(rc), n, t.data_ptr(), f.data_ptr() if f is not None else None,
        f.stride(0) if f is not None else 0, rtol, atol, rank.data_ptr(), ties.data_ptr(), ws.data_ptr(),
        ws.numel(), _stream(dev)))
    return rank, ties


def loss_dense(scores, labels, loss: str = "bce", offset: float = 0.0, return_rows: bool = False):
    """KgeLoss (sum) on a dense score matrix (loss.py:153-159 / :198-213)."""
    _require_cuda(scores, labels)
    lib, k = _lib.load(), _Keep()
    x = _f32_rows(scores)
    n, m = x.shape
    lab = _labels(k, labels)
    dev = x.device
    out = torch.empty((), dtype=torch.float32, device=dev)
    rows = torch.empty(n, dtype=torch.float32, device=dev) if return_rows else None
    nbytes = n * ((m + 4095) // 4096) * 5 * 4 + 4096
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_loss_dense(x.data_ptr(), x.stride(0), n, m, C.byref(lab), LOSS[loss], offset,
                                      out.data_ptr(), rows.data_ptr() if rows is not None else None,
                                      ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, rows) if return_rows else out


def rank_dense(scores, true_scores, filter_labels=None, rtol: float = 1e-4, atol: float = 1e-5,
               rank=None, ties=None):
    """_get_ranks_and_num_ties (+ optional filter subtraction) on dense scores; integer, bit-exact."""
    _require_cuda(scores, true_scores, filter_labels)
    lib = _lib.load()
    x = _f32_rows(scores)
    n, m = x.shape
    dev = x.device
    t = true_scores.reshape(-1).float().contiguous()
    if rank is None:
        rank = torch.zeros(n, dtype=torch.int64, device=dev)
    if ties is None:
        ties = torch.zeros(n, dtype=torch.int64, device=dev)
    f = None
    if filter_labels is not None:
        f = _f32_rows(filter_labels)
    _lib.check(lib.b200kge_rank_dense(x.data_ptr(), x.stride(0), n, m, t.data_ptr(),
                                      f.data_ptr() if f is not None else None,
                                      f.stride(0) if f is not None else 0, rtol, atol, rank.data_ptr(),
                                      ties.data_ptr(), _stream(dev)))
    return rank, ties


def ns_score(model: str, ent, rel, triples, negatives, slot: int, with_positive: bool = False,
             l_norm: float = 1.0, dropout: Optional["DropoutKey"] = None, implementation: str = "batch"):
    """[n, K] (or [n, 1+K] with the positive in column 0) negative-sample scores.

    With `dropout` (an engine.DropoutKey) the slot's six embedding-dropout draws are applied
    (b200kge_ns_score_dropout): `implementation` ("triple", "batch" or "all") selects how the negatives' masks are
    drawn, as the reference's negative_sampling.implementation does; the block always has the positive in column 0."""
    _require_cuda(ent, rel, triples, negatives)
    lib, k = _lib.load(), _Keep()
    if dropout is not None:
        if not with_positive:
            raise ValueError("ns_score with dropout returns the [n, 1+K] block (with_positive=True)")
        re_, rr = k.rows(ent), k.rows(rel)
        tri = _i64_block(triples)
        neg = _i64_block(negatives)
        n, K = neg.shape
        out = torch.empty((n, K + 1), dtype=torch.float32, device=ent.device)
        _lib.check(lib.b200kge_ns_score_dropout(MODELS[model], l_norm, C.byref(re_), C.byref(rr), tri.data_ptr(),
                                                int(slot), neg.data_ptr(), n, K, NS_IMPL[implementation],
                                                C.byref(dropout.struct()), out.data_ptr(), out.stride(0),
                                                _stream(ent.device)))
        return out
    tri = triples.long()
    rs, rp, ro = k.rows(ent, tri[:, S].contiguous()), k.rows(rel, tri[:, P].contiguous()), \
        k.rows(ent, tri[:, O].contiguous())
    neg = negatives.long().contiguous()
    n, K = neg.shape
    table = k.rows(rel if slot == P else ent)
    dev = ent.device
    out = torch.empty((n, K + (1 if with_positive else 0)), dtype=torch.float32, device=dev)
    _lib.check(lib.b200kge_ns_score(MODELS[model], l_norm, C.byref(rs), C.byref(rp), C.byref(ro),
                                    C.byref(table), slot, neg.data_ptr(), n, K, 1 if with_positive else 0,
                                    out.data_ptr(), out.stride(0), _stream(dev)))
    return out


def sample_uniform(n: int, K: int, vocab: int, seed: int, offset: int, device) -> torch.Tensor:
    """[n, K] int64 ids ~ U{0..vocab-1} drawn on the device (Philox4x32-10 keyed by seed, counter = (position, offset))."""
    lib = _lib.load()
    out = torch.empty((n, K), dtype=torch.int64, device=device)
    if not out.is_cuda:
        raise RuntimeError("kge_b200 runs on CUDA (sm_90) tensors only; there is no CPU path")
    _lib.check(lib.b200kge_sample_uniform(seed & (2 ** 64 - 1), offset & (2 ** 64 - 1), vocab, n, K, out.data_ptr(),
                                          _stream(out.device)))
    return out


class FilterIndex:
    """The positives of one negative-sampling slot, resident on `device`: keys [k,2], offsets [k+1], values [nnz] (int64,
    include/b200kge.h b200kge_filter_index_build) built once on the host from a KvsAllIndex (`dataset.index(...)` of the
    reference, or kge_b200.indexing's).  `max_count` is the largest number of distinct positives of one key."""

    def __init__(self, index, vocab: int, device):
        from .indexing import filter_csr

        keys, offsets, values, self.max_count = filter_csr(index, vocab)
        self.vocab = int(vocab)
        self.keys, self.offsets, self.values = (t.to(device) for t in (keys, offsets, values))

    def __len__(self) -> int:
        return self.keys.shape[0]


def sample_uniform_filtered(n: int, K: int, vocab: int, seed: int, offset: int, triples: torch.Tensor, slot: int,
                            index: FilterIndex) -> torch.Tensor:
    """[n, K] int64 ids ~ U({0..vocab-1} minus the positives of row i's key) drawn on the device; the key of row i of
    triples [n,3] is (p, o) for slot S, (s, o) for P, (s, p) for O.  Positions whose first draw is not a positive equal
    sample_uniform(n, K, vocab, seed, offset); rows whose positives cover the vocabulary get -1."""
    if index.vocab != vocab:
        raise ValueError(f"the filter index was built for a vocabulary of {index.vocab}, not {vocab}")
    _require_cuda(triples, index.keys)
    tri = _i64_block(triples)
    if tri.dim() != 2 or tri.shape[1] != 3 or tri.shape[0] != n:
        raise ValueError(f"expected triples [{n}, 3], got {tuple(tri.shape)}")
    out = torch.empty((n, K), dtype=torch.int64, device=tri.device)
    _lib.check(_lib.load().b200kge_sample_uniform_filtered(
        seed & (2 ** 64 - 1), offset & (2 ** 64 - 1), vocab, n, K, tri.data_ptr(), int(slot), index.keys.data_ptr(),
        index.offsets.data_ptr(), index.values.data_ptr(), len(index), out.data_ptr(), _stream(out.device)))
    return out


class FrequencyTable:
    """The weights of frequency sampling for one slot (KgeFrequencySampler, sampler.py:755-793): counts [V] per id (the
    slot's column of the training split, bincount'ed) plus `smoothing`, quantised once on the host to integer weights
    (indexing.frequency_cdf) and uploaded as their exclusive prefix `cdf` [V+1] (int64, cdf[V] = Q <= 2^62)."""

    def __init__(self, counts: torch.Tensor, smoothing: float, device):
        from .indexing import frequency_cdf

        cdf = frequency_cdf(counts, smoothing)
        self.vocab = cdf.numel() - 1
        self.smoothing = float(smoothing)
        self.total = int(cdf[-1])
        self.cdf = cdf.to(device)

    def attach(self, index: "FilterIndex") -> "FilterIndex":
        """Gives `index` the per-entry table of sample_frequency_filtered under these weights: `index.below` [nnz]
        (device), `index.full_keys` (number of keys whose positives carry all the weight, so that no negative exists
        for them) and `index.first_full_key` (its (a, b), or None).  Returns `index`."""
        from .indexing import frequency_below

        if index.vocab != self.vocab:
            raise ValueError(f"the filter index was built for a vocabulary of {index.vocab}, not {self.vocab}")
        below, full, first = frequency_below(self.cdf.cpu(), index.offsets.cpu(), index.values.cpu())
        index.below = below.to(index.values.device)
        index.below_table = self
        index.full_keys = full
        index.first_full_key = tuple(index.keys[first].tolist()) if first >= 0 else None
        return index


def sample_frequency(n: int, K: int, table: FrequencyTable, seed: int, offset: int) -> torch.Tensor:
    """[n, K] int64 ids drawn on the device with P(x) = q_x / Q, the quantised weights of `table`; each element takes the
    64-bit draw of sample_uniform(n, K, vocab, seed, offset) (equal weights reproduce it)."""
    _require_cuda(table.cdf)
    out = torch.empty((n, K), dtype=torch.int64, device=table.cdf.device)
    _lib.check(_lib.load().b200kge_sample_frequency(
        seed & (2 ** 64 - 1), offset & (2 ** 64 - 1), table.vocab, table.cdf.data_ptr(), n, K, out.data_ptr(),
        _stream(out.device)))
    return out


def sample_frequency_filtered(n: int, K: int, table: FrequencyTable, seed: int, offset: int, triples: torch.Tensor,
                              slot: int, index: FilterIndex) -> torch.Tensor:
    """[n, K] int64 ids drawn on the device with P(y) = q_y / (Q - M_i) over the ids y that are not positives of row i's
    key (M_i: the weight of its positives); keys as in sample_uniform_filtered, `index` attached to `table`
    (FrequencyTable.attach).  Positions whose first draw is not a positive equal sample_frequency(n, K, table, seed,
    offset); rows whose positives carry all the weight get -1."""
    if index.vocab != table.vocab:
        raise ValueError(f"the filter index was built for a vocabulary of {index.vocab}, not {table.vocab}")
    if getattr(index, "below_table", None) is not table:
        raise ValueError("the filter index is not attached to this frequency table (FrequencyTable.attach)")
    _require_cuda(triples, index.keys, table.cdf)
    tri = _i64_block(triples)
    if tri.dim() != 2 or tri.shape[1] != 3 or tri.shape[0] != n:
        raise ValueError(f"expected triples [{n}, 3], got {tuple(tri.shape)}")
    out = torch.empty((n, K), dtype=torch.int64, device=tri.device)
    _lib.check(_lib.load().b200kge_sample_frequency_filtered(
        seed & (2 ** 64 - 1), offset & (2 ** 64 - 1), table.vocab, n, K, tri.data_ptr(), int(slot),
        index.keys.data_ptr(), index.offsets.data_ptr(), index.values.data_ptr(), len(index), table.cdf.data_ptr(),
        index.below.data_ptr(), out.data_ptr(), _stream(out.device)))
    return out


def _train_1vsall_forward(model, ent, rel, triples, num_relations, loss, offset, l_norm, precision, dropout, out=None,
                          workspace=None):
    _require_cuda(ent, rel, triples)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri = _i64_block(triples)
    n = tri.shape[0]
    dev = ent.device
    if out is None:
        out = torch.empty((), dtype=torch.float32, device=dev)
    if dropout is not None:
        ws = torch.empty(lib.b200kge_train_1vsall_workspace_bytes(MODELS[model], n, ent.shape[0], ent.shape[1], 1),
                         dtype=torch.uint8, device=dev)
    else:
        ws = workspace if workspace is not None else _workspace(MODELS[model], n, ent.shape[0], ent.shape[1], False, dev)
    _lib.check(lib.b200kge_train_1vsall_forward(
        MODELS[model], l_norm, PREC[precision], C.byref(re_), C.byref(rr), int(num_relations), tri.data_ptr(), n,
        LOSS[loss], offset, None if dropout is None else C.byref(dropout.struct()), out.data_ptr(), ws.data_ptr(),
        ws.numel(), _stream(dev)))
    return out


def train_1vsall_forward(model: str, ent, rel, triples, loss: str = "bce", offset: float = 0.0,
                         l_norm: float = 1.0, precision: str = "auto", out=None, workspace=None,
                         dropout: Optional["DropoutKey"] = None):
    """One fused 1vsAll forward step for device-resident triples [n,3]; returns the 0-d loss
    (loss(score_sp,o) + loss(score_po,s)) / n  (train_1vsAll.py:48-82).  With `dropout` the six embedding-dropout draws
    of the step are applied (b200kge_train_1vsall_forward with a dropout key; `workspace` is not used)."""
    return _train_1vsall_forward(model, ent, rel, triples, 0, loss, offset, l_norm, precision, dropout, out, workspace)


class Step1vsAll:
    """A prepared fused 1vsAll forward step for device-resident batches: table views, enums, workspace and the
    output scalar are set up once, a call is ONE ctypes call (the job plugin's per-batch path; saves ~20 us of Python
    per step against train_1vsall_forward).  The returned 0-d tensor is a persistent buffer that the next call
    overwrites — read it (`.item()`) before calling again.  Valid as long as the tables keep their storage."""

    def __init__(self, model: str, ent: torch.Tensor, rel: torch.Tensor, max_n: int, loss: str = "bce",
                 offset: float = 0.0, l_norm: float = 1.0, precision: str = "auto"):
        _require_cuda(ent, rel)
        self.lib = _lib.load()
        self.ent, self.rel = _f32(ent), _f32(rel)
        self.k = _Keep()
        self.re, self.rr = self.k.rows(self.ent), self.k.rows(self.rel)
        self.max_n = int(max_n)
        nbytes = self.lib.b200kge_workspace_bytes(MODELS[model], self.max_n, ent.shape[0], ent.shape[1], 0)
        self.ws = torch.empty(nbytes + self.max_n * 24 + 1024, dtype=torch.uint8, device=ent.device)   # + staged batch (host form)
        self.out = torch.zeros((), dtype=torch.float32, device=ent.device)
        self.loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        self.loss_np = self.loss_host.numpy()
        self.key = (self.ent.data_ptr(), self.rel.data_ptr(), tuple(ent.shape), tuple(rel.shape))
        self.args = (MODELS[model], C.c_float(l_norm), PREC[precision], C.byref(self.re), C.byref(self.rr))
        self.loss_args = (LOSS[loss], C.c_float(offset))
        self.out_ptr = C.c_void_p(self.out.data_ptr())
        self.ws_args = (C.c_void_p(self.ws.data_ptr()), self.ws.numel())
        self.dev = ent.device

    def matches(self, ent, rel, n):
        return n <= self.max_n and self.key == (ent.data_ptr(), rel.data_ptr(), tuple(ent.shape), tuple(rel.shape))

    def __call__(self, triples: torch.Tensor) -> torch.Tensor:
        triples = _i64_block(triples)
        # plain model (num_relations = 0), no dropout
        rc = self.lib.b200kge_train_1vsall_forward(*self.args, 0, C.c_void_p(triples.data_ptr()), triples.shape[0],
                                                   *self.loss_args, None, self.out_ptr, *self.ws_args, _stream(self.dev))
        if rc:
            _lib.check(rc)
        return self.out

    def call_host(self, triples_host: torch.Tensor) -> float:
        """The same step from a HOST batch (contiguous int64 [n,3], ideally pinned): host->device copy, kernels, the
        4-byte read-back and the stream synchronisation inside ONE library call (triples.to(device) ... .item(),
        train_1vsAll.py:59-77)."""
        rc = self.lib.b200kge_train_1vsall_forward_host(
            *self.args, C.c_void_p(triples_host.data_ptr()), triples_host.shape[0], *self.loss_args,
            C.c_void_p(self.loss_host.data_ptr()), *self.ws_args, _stream(self.dev))
        if rc:
            _lib.check(rc)
        return float(self.loss_np[0])


class HostStep:
    """End-to-end 1vsAll forward step with HOST buffers (pinned in, scalar out): the call a
    training loop makes per batch — triples.to(device) ... loss.item() (train_1vsAll.py:59-77)."""

    def __init__(self, model: str, ent: torch.Tensor, rel: torch.Tensor, max_n: int, loss: str = "bce",
                 offset: float = 0.0, l_norm: float = 1.0, precision: str = "auto"):
        _require_cuda(ent, rel)
        self.model, self.loss, self.offset, self.l_norm, self.precision = model, loss, offset, l_norm, precision
        self.ent, self.rel = _f32(ent), _f32(rel)
        self.k = _Keep()
        self.re, self.rr = self.k.rows(self.ent), self.k.rows(self.rel)
        self.ws = _workspace(MODELS[model], max_n, ent.shape[0], ent.shape[1], False, ent.device)
        self.loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        self.h2d_bytes = 0
        self.d2h_bytes = 4

    def __call__(self, triples_host: torch.Tensor) -> float:
        if triples_host.is_cuda or triples_host.dtype != torch.int64 or not triples_host.is_contiguous():
            raise ValueError("triples_host must be a contiguous int64 CPU tensor [n,3]")
        n = triples_host.shape[0]
        self.h2d_bytes = n * 3 * 8
        _lib.check(_lib.load().b200kge_train_1vsall_forward_host(
            MODELS[self.model], self.l_norm, PREC[self.precision], C.byref(self.re), C.byref(self.rr),
            triples_host.data_ptr(), n, LOSS[self.loss], self.offset, self.loss_host.data_ptr(),
            self.ws.data_ptr(), self.ws.numel(), _stream(self.ent.device)))
        return float(self.loss_host[0])


# ---- SURVEY 8f rows (gradients, penalties, CSR labels) ---------------------------------------------------------
def gemm_nt(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """C = A @ B^T (fp32 in/out) on the f16 tensor pipe from pre-split hi/lo fp16 planes."""
    _require_cuda(a, b)
    lib = _lib.load()
    a, b = _f32(a), _f32(b)
    M, K = a.shape
    N = b.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    ws = torch.empty(lib.b200kge_gemm_nt_workspace_bytes(M, N, K), dtype=torch.uint8, device=a.device)
    _lib.check(lib.b200kge_gemm_nt(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, K, out.data_ptr(),
                                     out.stride(0), ws.data_ptr(), ws.numel(), _stream(a.device)))
    return out


def _train_1vsall_backward(model, ent, rel, triples, num_relations, loss, offset, l_norm, dropout):
    _require_cuda(ent, rel, triples)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri = _i64_block(triples)
    n = tri.shape[0]
    dev = ent.device
    d_ent = torch.empty_like(_f32(ent))
    d_rel = torch.empty_like(_f32(rel))
    nbytes = lib.b200kge_train_1vsall_workspace_bytes(MODELS[model], n, ent.shape[0], ent.shape[1],
                                                      0 if dropout is None else 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_train_1vsall_backward(
        MODELS[model], l_norm, C.byref(re_), C.byref(rr), int(num_relations), tri.data_ptr(), n, LOSS[loss], offset,
        None if dropout is None else C.byref(dropout.struct()), d_ent.data_ptr(), d_ent.stride(0), d_rel.data_ptr(),
        d_rel.stride(0), ws.data_ptr(), ws.numel(), _stream(dev)))
    return d_ent, d_rel


def train_1vsall_backward(model: str, ent, rel, triples, loss: str = "bce", offset: float = 0.0, l_norm: float = 1.0,
                          dropout: Optional["DropoutKey"] = None):
    """(d_ent, d_rel): dense table gradients of train_1vsall_forward's loss (dot family; TransE L1/L2; RotatE L1), with
    the forward's dropout masks when `dropout` is the forward's key."""
    return _train_1vsall_backward(model, ent, rel, triples, 0, loss, offset, l_norm, dropout)


def train_1vsall_reciprocal_forward(model: str, ent, rel, triples, num_relations: int, loss: str = "bce",
                                    offset: float = 0.0, l_norm: float = 1.0, precision: str = "auto",
                                    dropout: Optional["DropoutKey"] = None):
    """The 1vsAll step of a reciprocal-relations model (rel holds 2 * num_relations rows): 0-d
    (loss(score_sp(s, p), o) + loss(score_sp(o, p + R), s)) / n  (reciprocal_relations_model.py:85-92), with the
    embedding-dropout draws of `dropout` (direction 1 on the _po streams) — b200kge_train_1vsall_forward with
    num_relations > 0."""
    return _train_1vsall_forward(model, ent, rel, triples, num_relations, loss, offset, l_norm, precision, dropout)


def train_1vsall_reciprocal_backward(model: str, ent, rel, triples, num_relations: int, loss: str = "bce",
                                     offset: float = 0.0, l_norm: float = 1.0, dropout: Optional["DropoutKey"] = None):
    """(d_ent, d_rel): dense table gradients (all 2R relation rows) of train_1vsall_reciprocal_forward's loss, under the
    forward's masks when `dropout` is the forward's key (dot family; TransE L1/L2; RotatE L1)."""
    return _train_1vsall_backward(model, ent, rel, triples, num_relations, loss, offset, l_norm, dropout)


def score_1vsN_backward(model: str, combine: str, ent, rel, q, p, grad_scores, l_norm: float = 1.0):
    """(d_ent, d_rel) of a dense [n, E] score block given dL/dscores (fresh tensors): dot family (tensor cores), TransE
    L1 / L2 and RotatE L1 (row-gradient kernel)."""
    _require_cuda(ent, rel, grad_scores)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    qi, pi = _i64(q), _i64(p)
    g = _f32_rows(grad_scores)
    n = qi.numel()
    dev = ent.device
    d_ent = torch.empty_like(_f32(ent))
    d_rel = torch.empty_like(_f32(rel))
    ws = torch.empty(lib.b200kge_score_1vsN_backward_workspace_bytes(MODELS[model], n, ent.shape[0], ent.shape[1]),
                     dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_score_1vsN_backward(
        MODELS[model], SP_ if combine == "sp_" else _PO, l_norm, C.byref(re_), C.byref(rr), qi.data_ptr(), pi.data_ptr(), n,
        g.data_ptr(), g.stride(0), d_ent.data_ptr(), d_ent.stride(0), d_rel.data_ptr(), d_rel.stride(0), ws.data_ptr(),
        ws.numel(), _stream(dev)))
    return d_ent, d_rel


def score_1vsN_loss_csr_backward(model: str, combine: str, ent, rel, q, p, csr_offsets, csr_cols, loss: str = "kl",
                                 offset: float = 0.0, label_smoothing: float = 0.0, batch_size: Optional[int] = None,
                                 dropout: Optional["DropoutKey"] = None, dropout_streams: Optional[str] = None,
                                 l_norm: float = 1.0):
    """(d_ent, d_rel) of score_1vsN_loss_csr(...) / batch_size over the whole entity table (dot family; TransE with
    l_norm 1 or 2; RotatE with l_norm 1 — other norms raise NotImplementedError), with the forward's dropout masks when
    `dropout` is the forward's key (and `dropout_streams` the forward's)."""
    _require_cuda(ent, rel, csr_offsets, csr_cols)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    qi, pi, offs, cols = _i64(q), _i64(p), _i64(csr_offsets), _i64(csr_cols)
    n = qi.numel()
    dev = ent.device
    d_ent = torch.empty_like(_f32(ent))
    d_rel = torch.empty_like(_f32(rel))
    if dropout is not None:
        nbytes = lib.b200kge_score_1vsN_loss_csr_dropout_workspace_bytes(MODELS[model], n, ent.shape[0], ent.shape[1],
                                                                          int(cols.numel()))
    else:
        nbytes = lib.b200kge_score_1vsN_backward_workspace_bytes(MODELS[model], n, ent.shape[0], ent.shape[1])
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_score_1vsN_loss_csr_backward(
        MODELS[model], SP_ if combine == "sp_" else _PO, SP_ if (dropout_streams or combine) == "sp_" else _PO, l_norm,
        C.byref(re_), C.byref(rr), qi.data_ptr(), pi.data_ptr(), n, offs.data_ptr(),
        cols.data_ptr() if cols.numel() else None, label_smoothing, LOSS[loss], offset, batch_size or n,
        None if dropout is None else C.byref(dropout.struct()), d_ent.data_ptr(), d_ent.stride(0), d_rel.data_ptr(),
        d_rel.stride(0), ws.data_ptr(), ws.numel(), _stream(dev)))
    return d_ent, d_rel


def lookup_penalty(weight: torch.Tensor, regularize: str = "lp", regularize_weight: float = 0.0, p: float = 2.0,
                     weighted: bool = False, indexes: Optional[torch.Tensor] = None, space: str = "euclidean"):
    """LookupEmbedder.penalty (lookup_embedder.py:123-177) as a 0-d tensor."""
    _require_cuda(weight, indexes)
    dev = weight.device
    if regularize == "" or regularize_weight == 0.0:
        return torch.zeros((), dtype=torch.float32, device=dev)
    if regularize == "n3":
        p = 3.0
    elif regularize != "lp":
        raise ValueError(f"Invalid value regularize={regularize}")
    lib, k = _lib.load(), _Keep()
    if regularize == "n3" and space != "complex":
        # the reference accepts n3 only in complex space (lookup_embedder.py:29-34), so its signed-cube branch for
        # weighted n3 elsewhere (:158) is unreachable
        raise ValueError("Illegal value n3 for key regularize; allowed values are ['', 'lp'] (space is not complex)")
    complex_abs = 1 if regularize == "n3" else 0
    counts = None
    if weighted:
        uniq, cnt = torch.unique(indexes, return_counts=True)
        rows = k.rows(weight, uniq)
        counts = cnt.float().contiguous()
        scale = regularize_weight / p / indexes.shape[0]          # len(indexes): rows of the index block
    else:
        rows = k.rows(weight)
        scale = regularize_weight / p
    out = torch.empty((), dtype=torch.float32, device=dev)
    ws = torch.empty(((int(rows.rows) + 7) // 8 + 2) * 4, dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_lookup_penalty(C.byref(rows), counts.data_ptr() if counts is not None else None, p,
                                            complex_abs, scale, out.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)))
    return out


def normalize_rows_(weight: torch.Tensor, p: float) -> torch.Tensor:
    """In-place row normalisation to unit Lp norm (lookup_embedder.py:64-69)."""
    _require_cuda(weight)
    w = _f32(weight)
    if w.data_ptr() != weight.data_ptr():
        raise ValueError("normalisation is in place: pass a row-contiguous float32 matrix")
    _lib.check(_lib.load().b200kge_normalize_rows(w.data_ptr(), w.stride(0), w.shape[0], w.shape[1], p,
                                                    _stream(w.device)))
    return weight


def ns_backward(model: str, ent, rel, triples, negatives: dict, offset: float = 0.0, l_norm: float = 1.0,
                  batch_size: Optional[int] = None, grad_scores: Optional[dict] = None,
                  dropout: Optional["DropoutKey"] = None, implementation: str = "batch"):
    """(d_ent, d_rel) of one negative-sampling batch; negatives = {slot: [n, K] ids}, slots 0 (S), 2 (O).

    Without grad_scores the loss is BCE with `offset`, divided by batch_size.  With grad_scores = {slot: G}, G [n, 1+K]
    (positive first) is dL/dscores of each slot's block already scaled — e.g. the G of ns_loss(..., want_grad=True) —
    and `offset` / `batch_size` are not used: any loss of ns_loss trains through the same kernel.

    With `dropout` (the forward's engine.DropoutKey and `implementation`) the gradients go through the forward's masks
    (b200kge_ns_backward with a dropout key); grad_scores is then required."""
    _require_cuda(ent, rel, triples)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri = _i64_block(triples)
    n = tri.shape[0]
    dev = ent.device
    d_ent = torch.zeros_like(_f32(ent))
    d_rel = torch.zeros_like(_f32(rel))
    if dropout is not None and grad_scores is None:
        raise ValueError("ns_backward with dropout needs grad_scores (e.g. the G of ns_loss(..., want_grad=True))")
    nbytes = lib.b200kge_ns_backward_workspace_bytes(MODELS[model], n, 0, ent.shape[1], 0 if dropout is None else 1)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    drop = None if dropout is None else C.byref(dropout.struct())
    impl = 0 if dropout is None else NS_IMPL[implementation]
    for slot, neg in negatives.items():
        ng = _i64_block(neg)
        g = None
        if grad_scores is not None:
            g = grad_scores[slot]
            _require_cuda(g)
            if g.shape != (n, ng.shape[1] + 1):
                raise ValueError(f"grad_scores[{slot}] has shape {tuple(g.shape)}, expected {(n, ng.shape[1] + 1)}")
            g = _f32_rows(g)
            k.refs.append(g)
        _lib.check(lib.b200kge_ns_backward(
            MODELS[model], l_norm, C.byref(re_), C.byref(rr), tri.data_ptr(), int(slot), ng.data_ptr(), n, ng.shape[1],
            impl, drop, g.data_ptr() if g is not None else None, g.stride(0) if g is not None else 0, offset,
            batch_size or n, d_ent.data_ptr(), d_ent.stride(0), d_rel.data_ptr(), d_rel.stride(0), ws.data_ptr(),
            ws.numel(), _stream(dev)))
    return d_ent, d_rel


def ns_backward_sparse(model: str, ent, rel, triples, slot: int, negatives, offset: float = 0.0, l_norm: float = 1.0,
                       batch_size: Optional[int] = None, grad_scores=None, dropout: Optional["DropoutKey"] = None,
                       implementation: str = "batch", sparse=(True, True)):
    """(d_ent, d_rel) of one slot of a negative-sampling batch, as ns_backward, with each table's gradient in the layout
    of LibKGE's `lookup_embedder.sparse` (b200kge_ns_backward_sparse).  sparse = (entities, relations): a dense [V, D]
    tensor where False; where True a coalesced torch.sparse_coo_tensor over the rows the reference looks up for the slot
    (the positives' s and o and every sampled id; the positives' p), or over every row of the entity table for
    implementation "all", whose open slot goes through embed_all().  "all" draws the dropout masks of "batch".
    grad_scores is the slot's [n, 1+K] block (or None: BCE with `offset` / batch_size).  The two row counts are read
    back with one device-to-host copy."""
    _require_cuda(ent, rel, triples, negatives)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri, ng = _i64_block(triples), _i64_block(negatives)
    n, K = tri.shape[0], ng.shape[1]
    E, R, D = ent.shape[0], rel.shape[0], ent.shape[1]
    dev = ent.device
    if dropout is not None and grad_scores is None:
        raise ValueError("ns_backward_sparse with dropout needs grad_scores (e.g. the G of ns_loss(..., want_grad=True))")
    g = None
    if grad_scores is not None:
        _require_cuda(grad_scores)
        if grad_scores.shape != (n, K + 1):
            raise ValueError(f"grad_scores has shape {tuple(grad_scores.shape)}, expected {(n, K + 1)}")
        g = _f32_rows(grad_scores)
    # embed_all() looks up every entity row: the dense gradient is the value block of the full row set
    ent_rows_all = sparse[0] and implementation == "all"
    flags = (int(sparse[0] and not ent_rows_all), int(sparse[1]))
    caps = (min(E, n * (K + 2)), min(R, n))
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    outs = []
    for f, tab, cap in ((flags[0], ent, caps[0]), (flags[1], rel, caps[1])):
        if f:
            outs.append((torch.empty(cap, dtype=torch.int64, device=dev),
                         torch.empty((cap, tab.shape[1]), dtype=torch.float32, device=dev)))
        else:
            outs.append((None, torch.zeros_like(_f32(tab))))
    (er, ev), (rr_, rv) = outs
    nbytes = lib.b200kge_ns_backward_sparse_workspace_bytes(MODELS[model], n, K, D, E, R, 0 if dropout is None else 1)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_ns_backward_sparse(
        MODELS[model], l_norm, C.byref(re_), C.byref(rr), tri.data_ptr(), int(slot), ng.data_ptr(), n, K,
        0 if dropout is None else NS_IMPL[implementation],
        None if dropout is None else C.byref(dropout.struct()), g.data_ptr() if g is not None else None,
        g.stride(0) if g is not None else 0, offset, batch_size or n,
        flags[0], er.data_ptr() if flags[0] else None, counts.data_ptr() if flags[0] else None, ev.data_ptr(),
        ev.stride(0), flags[1], rr_.data_ptr() if flags[1] else None, counts[1:].data_ptr() if flags[1] else None,
        rv.data_ptr(), rv.stride(0), ws.data_ptr(), ws.numel(), _stream(dev)))
    u = counts.tolist() if (flags[0] or flags[1]) else (0, 0)

    def layout(flag, rows, vals, V, want_sparse, u_):
        if flag:
            return torch.sparse_coo_tensor(rows[None, :u_], vals[:u_], (V, vals.shape[1]), is_coalesced=True)
        if want_sparse:       # "all": every row
            return torch.sparse_coo_tensor(torch.arange(V, device=dev)[None, :], vals, vals.shape, is_coalesced=True)
        return vals
    return (layout(flags[0], er, ev, E, ent_rows_all, u[0]), layout(flags[1], rr_, rv, R, False, u[1]))


def ns_p_backward(model: str, ent, rel, triples, negatives, grad_scores, l_norm: float = 1.0,
                  implementation: str = "batch", sparse=(False, False)):
    """(d_ent, d_rel) of the P slot of a negative-sampling batch (b200kge_ns_p_backward): triples [n, 3], negatives
    [n, K] relation ids, grad_scores = dL/dscores of the [n, 1+K] block (positive first), e.g. the G of
    ns_loss(..., want_grad=True).  sparse = (entities, relations) as in ns_backward_sparse: a dense [V, D] tensor where
    False; where True a coalesced torch.sparse_coo_tensor over the rows the reference looks up for the slot (the
    positives' s and o; the positives' p and every sampled id, or every relation row for implementation "all", whose
    score_so goes through embed_all()).  Raises NotImplementedError for an unserved model or norm and for more than
    NS_P_MAX_RELATIONS relations."""
    _require_cuda(ent, rel, triples, negatives, grad_scores)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri, ng = _i64_block(triples), _i64_block(negatives)
    n, K = tri.shape[0], ng.shape[1]
    E, R, D = ent.shape[0], rel.shape[0], ent.shape[1]
    dev = ent.device
    if grad_scores.shape != (n, K + 1):
        raise ValueError(f"grad_scores has shape {tuple(grad_scores.shape)}, expected {(n, K + 1)}")
    g = _f32_rows(grad_scores)
    rel_rows_all = sparse[1] and implementation == "all"
    flags = (int(sparse[0]), int(sparse[1] and not rel_rows_all))
    caps = (min(E, 2 * n), min(R, n * (K + 1)))
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    outs = []
    for f, tab, cap in ((flags[0], ent, caps[0]), (flags[1], rel, caps[1])):
        if f:
            outs.append((torch.empty(cap, dtype=torch.int64, device=dev),
                         torch.empty((cap, tab.shape[1]), dtype=torch.float32, device=dev)))
        else:
            outs.append((None, torch.zeros_like(_f32(tab))))
    (er, ev), (rr_, rv) = outs
    nbytes = lib.b200kge_ns_p_backward_workspace_bytes(MODELS[model], n, K, D, E, R)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_ns_p_backward(
        MODELS[model], l_norm, C.byref(re_), C.byref(rr), tri.data_ptr(), ng.data_ptr(), n, K, g.data_ptr(),
        g.stride(0), flags[0], er.data_ptr() if flags[0] else None, counts.data_ptr() if flags[0] else None,
        ev.data_ptr(), ev.stride(0), flags[1], rr_.data_ptr() if flags[1] else None,
        counts[1:].data_ptr() if flags[1] else None, rv.data_ptr(), rv.stride(0), ws.data_ptr(), ws.numel(),
        _stream(dev)))
    u = counts.tolist() if (flags[0] or flags[1]) else (0, 0)

    def layout(flag, rows, vals, V, want_sparse, u_):
        if flag:
            return torch.sparse_coo_tensor(rows[None, :u_], vals[:u_], (V, vals.shape[1]), is_coalesced=True)
        if want_sparse:       # "all": every relation row
            return torch.sparse_coo_tensor(torch.arange(V, device=dev)[None, :], vals, vals.shape, is_coalesced=True)
        return vals
    return (layout(flags[0], er, ev, E, False, u[0]), layout(flags[1], rr_, rv, R, rel_rows_all, u[1]))


def _shared_operands(unique, repeat, drop, n: int, K: int):
    """unique [U'], repeat [K - U] and drop [n] (None: "naive") of a shared sample as contiguous int64 device blocks."""
    un = _i64(unique)
    rp = _i64(repeat) if repeat is not None and repeat.numel() else None
    dr = _i64(drop) if drop is not None else None
    if dr is not None and dr.numel() != n:
        raise ValueError(f"drop has {dr.numel()} entries, expected one per row ({n})")
    U = un.numel() - (1 if dr is not None else 0)
    if K - U != (rp.numel() if rp is not None else 0):
        raise ValueError(f"repeat has {0 if rp is None else rp.numel()} entries, expected K - U = {K - U}")
    return un, rp, dr


def ns_shared_score(model: str, ent, rel, triples, slot: int, unique, repeat, drop, K: int, l_norm: float = 1.0,
                    precision: str = "auto", implementation: str = "batch", want_z: bool = False):
    """The [n, 1+K] block of one slot (0 = S, 2 = O) under shared negative sampling (b200kge_ns_shared_score): column 0
    the positive triple, column 1 + c the score of the shared id unique[u(i, c)] with j = c < U ? c : repeat[c - U] and
    u = j, or U where j == drop[i] ("default"; drop None: "naive").  unique, repeat and drop are the shared sample's
    _unique_samples, _repeat_indexes and the sub-batch's rows of _drop_index (sampler.py:383-585).  `implementation`
    "triple" adds F.pairwise_distance's eps to TransE's negatives.  want_z: also return Z [n, U'], the scores against
    the shared rows (the backward of TransE l_norm 2 needs them)."""
    _require_cuda(ent, rel, triples, unique)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri = _i64_block(triples)
    n = tri.shape[0]
    un, rp, dr = _shared_operands(unique, repeat, drop, n, K)
    dev = ent.device
    out = torch.empty((n, K + 1), dtype=torch.float32, device=dev)
    z = torch.empty((n, max(un.numel(), 1)), dtype=torch.float32, device=dev) if want_z else None
    nbytes = lib.b200kge_ns_shared_score_workspace_bytes(MODELS[model], n, un.numel(), ent.shape[1])
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_ns_shared_score(
        MODELS[model], l_norm, PREC[precision], C.byref(re_), C.byref(rr), tri.data_ptr(), int(slot), un.data_ptr(),
        un.numel(), rp.data_ptr() if rp is not None else None, dr.data_ptr() if dr is not None else None, n, K,
        NS_IMPL[implementation], out.data_ptr(), out.stride(0), z.data_ptr() if want_z else None,
        z.stride(0) if want_z else 0, ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, z[:, :un.numel()]) if want_z else out


def ns_shared_backward(model: str, ent, rel, triples, slot: int, unique, repeat, drop, K: int, grad_scores, z=None,
                       l_norm: float = 1.0, implementation: str = "batch", sparse=(False, False)):
    """(d_ent, d_rel) of ns_shared_score's block (b200kge_ns_shared_backward) for grad_scores = dL/dscores [n, 1+K],
    e.g. the G of ns_loss(..., want_grad=True); z is ns_shared_score's Z (required for TransE l_norm 2).  sparse =
    (entities, relations) as in ns_backward_sparse: where True a coalesced torch.sparse_coo_tensor over the rows the
    reference looks up for the slot (the positives' s and o with every shared id for "batch", the shared ids the rows
    use for "triple", every entity row for "all"; the positives' p)."""
    _require_cuda(ent, rel, triples, unique, grad_scores)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    tri = _i64_block(triples)
    n = tri.shape[0]
    un, rp, dr = _shared_operands(unique, repeat, drop, n, K)
    E, R, D = ent.shape[0], rel.shape[0], ent.shape[1]
    dev = ent.device
    if grad_scores.shape != (n, K + 1):
        raise ValueError(f"grad_scores has shape {tuple(grad_scores.shape)}, expected {(n, K + 1)}")
    g = _f32_rows(grad_scores)
    zz = _f32_rows(z) if z is not None else None
    ent_rows_all = sparse[0] and implementation == "all"
    flags = (int(sparse[0] and not ent_rows_all), int(sparse[1]))
    caps = (min(E, 2 * n + un.numel()), min(R, n))
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    outs = []
    for f, tab, cap in ((flags[0], ent, caps[0]), (flags[1], rel, caps[1])):
        if f:
            outs.append((torch.empty(cap, dtype=torch.int64, device=dev),
                         torch.empty((cap, tab.shape[1]), dtype=torch.float32, device=dev)))
        else:
            outs.append((None, torch.zeros_like(_f32(tab))))
    (er, ev), (rr_, rv) = outs
    nbytes = lib.b200kge_ns_shared_backward_workspace_bytes(MODELS[model], n, un.numel(), D, E, R)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_ns_shared_backward(
        MODELS[model], l_norm, C.byref(re_), C.byref(rr), tri.data_ptr(), int(slot), un.data_ptr(), un.numel(),
        rp.data_ptr() if rp is not None else None, dr.data_ptr() if dr is not None else None, n, K,
        NS_IMPL[implementation], zz.data_ptr() if zz is not None else None, zz.stride(0) if zz is not None else 0,
        g.data_ptr(), g.stride(0), flags[0], er.data_ptr() if flags[0] else None,
        counts.data_ptr() if flags[0] else None, ev.data_ptr(), ev.stride(0), flags[1],
        rr_.data_ptr() if flags[1] else None, counts[1:].data_ptr() if flags[1] else None, rv.data_ptr(),
        rv.stride(0), ws.data_ptr(), ws.numel(), _stream(dev)))
    u = counts.tolist() if (flags[0] or flags[1]) else (0, 0)

    def layout(flag, rows, vals, V, want_sparse, u_):
        if flag:
            return torch.sparse_coo_tensor(rows[None, :u_], vals[:u_], (V, vals.shape[1]), is_coalesced=True)
        if want_sparse:       # "all": every entity row
            return torch.sparse_coo_tensor(torch.arange(V, device=dev)[None, :], vals, vals.shape, is_coalesced=True)
        return vals
    return (layout(flags[0], er, ev, E, ent_rows_all, u[0]), layout(flags[1], rr_, rv, R, False, u[1]))


def ns_loss(scores, loss: str, arg: float = 0.0, temperature: float = 1.0, label_idx=None,
            batch_size: Optional[int] = None, want_grad: bool = False, return_rows: bool = False):
    """KgeLoss of a negative-sampling block (train_negative_sampling.py:126-156): scores [n, m] with one positive per
    row at label_idx[i] (None: column 0, the ns_score(with_positive=True) layout), label 0 elsewhere.  `loss` is any
    `train.loss` of the reference but ce; `arg` is the offset (bce, bce_mean, bce_self_adversarial) or the margin
    (margin_ranking), `temperature` that of bce_self_adversarial.

    Returns (loss, G): loss = sum of the row losses / batch_size (0-d tensor, deterministic); G = dL/dscores [n, m]
    (fp32) when want_grad, else None.  With return_rows the per-row losses (not divided) follow as a third item."""
    _require_cuda(scores, label_idx)
    if loss not in LOSS:
        raise ValueError(f"unknown loss {loss!r}")
    lib = _lib.load()
    x = scores if (scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1) \
        else scores.float().contiguous()
    n, m = x.shape
    dev = x.device
    li = _i64(label_idx)
    if li is not None and li.numel() != n:
        raise ValueError(f"label_idx has {li.numel()} entries for {n} rows")
    out = torch.empty((), dtype=torch.float32, device=dev)
    G = torch.empty((n, m), dtype=torch.float32, device=dev) if want_grad else None
    rows = torch.empty(n, dtype=torch.float32, device=dev) if return_rows else None
    ws = torch.empty(lib.b200kge_ns_loss_workspace_bytes(n), dtype=torch.uint8, device=dev)
    scale = 1.0 / float(batch_size) if batch_size else 1.0
    _lib.check(lib.b200kge_ns_loss(
        x.data_ptr(), x.stride(0), n, m, li.data_ptr() if li is not None else None, LOSS[loss], float(arg),
        float(temperature), scale, out.data_ptr(), rows.data_ptr() if rows is not None else None,
        G.data_ptr() if G is not None else None, m, ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, G, rows) if return_rows else (out, G)


def score_1vsN_loss_csr(model: str, combine: str, q_tab, rel, cand_tab, csr_offsets, csr_cols, q=None, p=None,
                          loss: str = "kl", offset: float = 0.0, label_smoothing: float = 0.0, l_norm: float = 1.0,
                          precision: str = "auto", return_rows: bool = False, dropout: Optional["DropoutKey"] = None,
                          dropout_streams: Optional[str] = None):
    """KvsAll loss (sum over rows) with CSR multi-hot labels — see b200kge_score_1vsN_loss_csr.  With `dropout` the three
    embedding-dropout draws of the query type are applied (b200kge_score_1vsN_loss_csr_dropout): the queries are rows
    q of the entity table q_tab, which must also be the candidate table.  `dropout_streams` ("sp_" | "_po") draws the
    masks of that query type instead of `combine`'s (a reciprocal-relations model's _po queries: combine "sp_",
    streams "_po": the `mask_dir` of b200kge_score_1vsN_loss_csr_dropout)."""
    _require_cuda(q_tab, rel, cand_tab, csr_offsets, csr_cols)
    lib, k = _lib.load(), _Keep()
    rq, rp, rc = k.rows(q_tab, q), k.rows(rel, p), k.rows(cand_tab)
    n, m = int(rq.rows), int(rc.rows)
    dev = q_tab.device
    offs, cols = _i64(csr_offsets), _i64(csr_cols)
    nnz = int(cols.numel())
    out = torch.empty((), dtype=torch.float32, device=dev)
    rows = torch.empty(n, dtype=torch.float32, device=dev) if return_rows else None
    if dropout is not None:
        if q is None or p is None or q_tab.data_ptr() != cand_tab.data_ptr():
            raise ValueError("dropout needs query indexes into the candidate table (q_tab is cand_tab) and relation indexes")
        re_, rr = k.rows(cand_tab), k.rows(rel)
        qi, pi = _i64(q), _i64(p)
        k.refs += [qi, pi]
        ws = torch.empty(lib.b200kge_score_1vsN_loss_csr_dropout_workspace_bytes(MODELS[model], n, m, rq.dim, nnz),
                         dtype=torch.uint8, device=dev)
        _lib.check(lib.b200kge_score_1vsN_loss_csr_dropout(
            MODELS[model], SP_ if combine == "sp_" else _PO, SP_ if (dropout_streams or combine) == "sp_" else _PO,
            l_norm, PREC[precision], C.byref(re_), C.byref(rr), qi.data_ptr(), pi.data_ptr(), n, offs.data_ptr(),
            cols.data_ptr() if nnz else None, nnz, label_smoothing, LOSS[loss], offset, C.byref(dropout.struct()),
            out.data_ptr(), rows.data_ptr() if rows is not None else None, ws.data_ptr(), ws.numel(), _stream(dev)))
        return (out, rows) if return_rows else out
    nbytes = lib.b200kge_score_1vsN_loss_csr_workspace_bytes(MODELS[model], n, m, rq.dim, nnz)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.b200kge_score_1vsN_loss_csr(
        MODELS[model], SP_ if combine == "sp_" else _PO, l_norm, PREC[precision], C.byref(rq), C.byref(rp), C.byref(rc),
        n, offs.data_ptr(), cols.data_ptr() if nnz else None, nnz, label_smoothing, LOSS[loss], offset, out.data_ptr(),
        rows.data_ptr() if rows is not None else None, ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, rows) if return_rows else out


def _so_workspace(lib, model, n, ent, rel, nnz, dropout, dev) -> torch.Tensor:
    return torch.empty(lib.b200kge_score_so_loss_csr_workspace_bytes(MODELS[model], n, rel.shape[0], ent.shape[1], nnz,
                                                                     0 if dropout is None else 1),
                       dtype=torch.uint8, device=dev)


def score_so_loss_csr(model: str, ent, rel, s, o, csr_offsets, csr_cols, loss: str = "kl", offset: float = 0.0,
                      precision: str = "auto", return_rows: bool = False, dropout: Optional["DropoutKey"] = None):
    """KvsAll loss of the s_o query type (sum over rows; relation prediction, train_KvsAll.py:251-254 with score_so): the
    pairs (ent[s_i], ent[o_i]) against every relation, CSR labels = relation ids, no label smoothing.  With `dropout`
    the three s_o draws (streams 24-26) are applied.  See b200kge_score_so_loss_csr; the dot family only."""
    _require_cuda(ent, rel, csr_offsets, csr_cols)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    si, oi, offs, cols = _i64(s), _i64(o), _i64(csr_offsets), _i64(csr_cols)
    n, nnz = si.numel(), int(cols.numel())
    dev = ent.device
    out = torch.empty((), dtype=torch.float32, device=dev)
    rows = torch.empty(n, dtype=torch.float32, device=dev) if return_rows else None
    ws = _so_workspace(lib, model, n, ent, rel, nnz, dropout, dev)
    _lib.check(lib.b200kge_score_so_loss_csr(
        MODELS[model], 1.0, PREC[precision], C.byref(re_), C.byref(rr), si.data_ptr(), oi.data_ptr(), n, offs.data_ptr(),
        cols.data_ptr() if nnz else None, nnz, LOSS[loss], offset, None if dropout is None else C.byref(dropout.struct()),
        out.data_ptr(), rows.data_ptr() if rows is not None else None, ws.data_ptr(), ws.numel(), _stream(dev)))
    return (out, rows) if return_rows else out


def score_so_loss_csr_backward(model: str, ent, rel, s, o, csr_offsets, csr_cols, loss: str = "kl",
                               offset: float = 0.0, batch_size: Optional[int] = None,
                               dropout: Optional["DropoutKey"] = None):
    """(d_ent, d_rel) of score_so_loss_csr(...) / batch_size (fresh tensors), with the forward's dropout masks when
    `dropout` is the forward's key."""
    _require_cuda(ent, rel, csr_offsets, csr_cols)
    lib, k = _lib.load(), _Keep()
    re_, rr = k.rows(ent), k.rows(rel)
    si, oi, offs, cols = _i64(s), _i64(o), _i64(csr_offsets), _i64(csr_cols)
    n = si.numel()
    dev = ent.device
    d_ent = torch.empty_like(_f32(ent))
    d_rel = torch.empty_like(_f32(rel))
    ws = _so_workspace(lib, model, n, ent, rel, int(cols.numel()), dropout, dev)
    _lib.check(lib.b200kge_score_so_loss_csr_backward(
        MODELS[model], 1.0, C.byref(re_), C.byref(rr), si.data_ptr(), oi.data_ptr(), n, offs.data_ptr(),
        cols.data_ptr() if cols.numel() else None, LOSS[loss], offset, batch_size or n,
        None if dropout is None else C.byref(dropout.struct()), d_ent.data_ptr(), d_ent.stride(0), d_rel.data_ptr(),
        d_rel.stride(0), ws.data_ptr(), ws.numel(), _stream(dev)))
    return d_ent, d_rel


def _optim_operands(param, state, grad):
    """(rows, dim, grad values, grad row ids or None, nnz, coalesced) of one optimizer step: param and its state as
    contiguous fp32 CUDA tensors viewed [rows, dim], the gradient dense or a COO tensor with one sparse dimension."""
    _require_cuda(param, grad, *state)
    for t in (param, *state):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.layout != torch.strided:
            raise TypeError("the optimizer step takes contiguous float32 parameters and state")
        if t.shape != param.shape:
            raise ValueError(f"state of shape {tuple(t.shape)} for a parameter of shape {tuple(param.shape)}")
    if grad.shape != param.shape:
        raise ValueError(f"gradient of shape {tuple(grad.shape)} for a parameter of shape {tuple(param.shape)}")
    rows = param.shape[0] if param.dim() > 0 and param.numel() > 0 else (1 if param.numel() else 0)
    dim = param.numel() // rows if rows > 0 else 1
    if not grad.is_sparse:
        g = grad if (grad.dtype == torch.float32 and grad.is_contiguous()) else grad.float().contiguous()
        return rows, dim, g, None, 0, 1
    if grad.sparse_dim() != 1:
        raise NotImplementedError(f"a sparse gradient with {grad.sparse_dim()} sparse dimensions (the optimizer step "
                                  "takes row-sparse gradients: one sparse dimension)")
    idx, vals = grad._indices()[0], grad._values()
    idx = idx if idx.is_contiguous() else idx.contiguous()
    vals = vals if (vals.dtype == torch.float32 and vals.is_contiguous()) else vals.float().contiguous()
    return rows, dim, vals, idx, idx.numel(), int(grad.is_coalesced())


def _optim_workspace(lib, rows, dim, nnz, coalesced, idx, dev):
    nbytes = lib.b200kge_optim_step_workspace_bytes(rows, dim, nnz, coalesced) if idx is not None else 0
    return torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None


def adagrad_step(param, state_sum, grad, clr: float, eps: float, weight_decay: float = 0.0,
                 foreach_order: bool = True) -> None:
    """One parameter of torch.optim.Adagrad.step() in place (b200kge_adagrad_step): param and state_sum (the state's
    "sum") are updated with grad, dense or a torch.sparse_coo_tensor of value rows, coalesced or not.  clr is
    lr / (1 + (step - 1) lr_decay) after the step count was incremented; foreach_order selects the order of torch's
    _multi_tensor_adagrad (True) or _single_tensor_adagrad (False) for a dense gradient.  Runs on the parameter's
    current stream; the workspace of an uncoalesced gradient comes from torch's caching allocator."""
    lib = _lib.load()
    rows, dim, g, idx, nnz, coalesced = _optim_operands(param, (state_sum,), grad)
    if rows * dim == 0 or (idx is not None and nnz == 0):
        return
    ws = _optim_workspace(lib, rows, dim, nnz, coalesced, idx, param.device)
    _lib.check(lib.b200kge_adagrad_step(
        param.data_ptr(), state_sum.data_ptr(), rows, dim, g.data_ptr(), None if idx is None else idx.data_ptr(), nnz,
        coalesced, int(bool(foreach_order)), float(clr), float(eps), float(weight_decay),
        None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(), _stream(param.device)))


def sparse_adam_step(param, exp_avg, exp_avg_sq, grad, beta1: float, beta2: float, eps: float,
                     step_size: float) -> None:
    """One parameter of torch.optim.SparseAdam.step() in place (b200kge_sparse_adam_step) with a torch.sparse_coo_tensor
    gradient, coalesced or not: step_size = lr sqrt(1 - beta2^t) / (1 - beta1^t) after the step count t was
    incremented.  1 - beta is formed here in double precision, as torch forms it."""
    lib = _lib.load()
    if not grad.is_sparse:
        raise RuntimeError("SparseAdam does not support dense gradients, please consider Adam instead")
    rows, dim, g, idx, nnz, coalesced = _optim_operands(param, (exp_avg, exp_avg_sq), grad)
    if rows * dim == 0 or nnz == 0:
        return
    ws = _optim_workspace(lib, rows, dim, nnz, coalesced, idx, param.device)
    _lib.check(lib.b200kge_sparse_adam_step(
        param.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(), rows, dim, g.data_ptr(), idx.data_ptr(), nnz,
        coalesced, float(1.0 - beta1), float(1.0 - beta2), float(eps), float(step_size),
        None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(), _stream(param.device)))
