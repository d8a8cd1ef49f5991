"""TEST INFRASTRUCTURE: CPU mirror of the embedding-dropout masks of libb200kge (kge_b200/csrc/dropout.cu, layout in
include/b200kge.h), the masked reference expressions of the 1vsAll and KvsAll steps in fp32 / fp64, engine stand-ins
that apply the mirror's masks (an extension of tests/engine_stub.py), and dropout modules that make the REFERENCE job
draw the mirror's masks instead of torch's."""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch

import engine_stub
from oracle import kge_oracle as orc
from philox_ref import MASK, philox4x32_10

SP_ENT, SP_REL, SP_TABLE, PO_TABLE, PO_REL, PO_ENT = range(6)
# (query entity, relation, table) streams of the sp_ (0) and _po (1) directions
DIR_STREAMS = ((SP_ENT, SP_REL, SP_TABLE), (PO_ENT, PO_REL, PO_TABLE))


def threshold(p):
    return int(math.floor((1.0 - float(np.float32(p))) * 4294967296.0))


def scale(p):
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def mask(p, seed, call, stream, rows, dim, row_base=0):
    """Keep mask [rows, dim] (bool) of draw `stream` over global rows [row_base, row_base + rows)."""
    th = threshold(p)
    e_lo, e_hi = row_base * dim, (row_base + rows) * dim
    out = np.zeros(rows * dim, dtype=bool)
    if rows * dim == 0:
        return torch.from_numpy(out.reshape(rows, dim))
    key = (seed & MASK, (seed >> 32) & MASK)
    for g in range(e_lo >> 2, ((e_hi - 1) >> 2) + 1):
        hi = (stream << 46) | g
        w = philox4x32_10([hi & MASK, (hi >> 32) & MASK, call & MASK, (call >> 32) & MASK], key)
        for j in range(4):
            e = 4 * g + j
            if e_lo <= e < e_hi:
                out[e - e_lo] = w[j] < th
    return torch.from_numpy(out.reshape(rows, dim))


def apply(x, p, seed, call, stream, row_base=0):
    """x with the draw's mask applied and kept values scaled by float32(1 / (1 - p)), in x's dtype."""
    if p == 0:
        return x
    m = mask(p, seed, call, stream, x.shape[0], x.shape[1], row_base).to(x.device)
    return torch.where(m, x * scale(p), torch.zeros((), dtype=x.dtype, device=x.device))


def _direction(model, ent, rel, a, p, key, direction, l_norm):
    """Scores [n, E] of one direction under its three draws (a: query entity ids, p: relation ids)."""
    sq, sr, st = DIR_STREAMS[direction]
    q = apply(ent[a], key.p_ent, key.seed, key.call, sq, key.row_base)
    r = apply(rel[p], key.p_rel, key.seed, key.call, sr, key.row_base)
    t = apply(ent, key.p_ent, key.seed, key.call, st, 0)
    if direction == 0:
        return orc.score_emb(model, q, r, t, "sp_", l_norm)
    return orc.score_emb(model, t, r, q, "_po", l_norm)


def loss_1vsall(model, ent, rel, triples, loss, offset, key, l_norm=1.0):
    """(loss(score_sp, o) + loss(score_po, s)) / n with the six draws of `key` (differentiable in ent / rel)."""
    triples = triples.long()
    s, p, o = triples[:, 0], triples[:, 1], triples[:, 2]
    total = 0.0
    for direction, a, lab in ((0, s, o), (1, o, s)):
        x = _direction(model, ent, rel, a, p, key, direction, l_norm)
        total = total + (orc.bce_loss(x, lab, offset) if loss == "bce" else orc.kl_loss(x, lab))
    return total / triples.shape[0]


def loss_kvsall(model, combine, ent, rel, q, p, offs, cols, loss, offset, label_smoothing, key, l_norm=1.0):
    """Sum over rows of the KvsAll loss of one query type with CSR labels under the draws of `key`."""
    x = _direction(model, ent, rel, q.long(), p.long(), key, 0 if combine == "sp_" else 1, l_norm)
    n, m = x.shape
    y = torch.zeros((n, m), dtype=x.dtype)
    counts = (offs[1:] - offs[:-1]).cpu()
    rows = torch.repeat_interleave(torch.arange(n), counts)
    y.index_put_((rows, cols.long().cpu()), torch.ones(len(rows), dtype=x.dtype), accumulate=True)
    if label_smoothing > 0:
        y = orc.kvsall_smooth_labels(y, label_smoothing)
    y = y.to(x.device)
    return orc.bce_loss(x, y, offset) if loss == "bce" else orc.kl_loss(x, y)


def grads(fn, ent, rel):
    e, r = ent.detach().clone().requires_grad_(True), rel.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        val = fn(e, r)
        de, dr = torch.autograd.grad(val, (e, r))
    return val.detach(), de, dr


# ---- engine stand-ins (CPU) that accept a dropout key ----------------------------------------------------------
calls = {"dropout": 0}


def _train_1vsall_forward(model, ent, rel, triples, loss="bce", offset=0.0, l_norm=1.0, precision="auto", out=None,
                          workspace=None, dropout=None):
    if dropout is None:
        return orc.train_1vsall_forward(model, ent, rel, triples.long(), loss, offset, l_norm)
    calls["dropout"] += 1
    return loss_1vsall(model, ent, rel, triples, loss, offset, dropout, l_norm)


def _train_1vsall_backward(model, ent, rel, triples, loss="bce", offset=0.0, l_norm=1.0, dropout=None):
    if dropout is None:
        return engine_stub.train_1vsall_backward(model, ent, rel, triples, loss, offset, l_norm)
    calls["dropout"] += 1
    return grads(lambda e, r: loss_1vsall(model, e, r, triples, loss, offset, dropout, l_norm), ent, rel)[1:]


def _score_1vsN_loss_csr(model, combine, q_tab, rel, cand_tab, csr_offsets, csr_cols, q=None, p=None, loss="kl",
                         offset=0.0, label_smoothing=0.0, l_norm=1.0, precision="auto", return_rows=False, dropout=None):
    if dropout is None:
        return engine_stub.score_1vsN_loss_csr(model, combine, q_tab, rel, cand_tab, csr_offsets, csr_cols, q, p, loss,
                                               offset, label_smoothing, l_norm, precision, return_rows)
    calls["dropout"] += 1
    return loss_kvsall(model, combine, cand_tab, rel, q, p, csr_offsets, csr_cols, loss, offset, label_smoothing,
                       dropout, l_norm)


def _score_1vsN_loss_csr_backward(model, combine, ent, rel, q, p, csr_offsets, csr_cols, loss="kl", offset=0.0,
                                  label_smoothing=0.0, batch_size=None, dropout=None):
    if dropout is None:
        return engine_stub.score_1vsN_loss_csr_backward(model, combine, ent, rel, q, p, csr_offsets, csr_cols, loss,
                                                        offset, label_smoothing, batch_size)
    calls["dropout"] += 1
    bs = batch_size or q.numel()
    return grads(lambda e, r: loss_kvsall(model, combine, e, r, q, p, csr_offsets, csr_cols, loss, offset,
                                          label_smoothing, dropout) / bs, ent, rel)[1:]


@contextlib.contextmanager
def installed():
    """engine_stub.installed() plus stand-ins of the four engine calls that take a dropout key; calls["dropout"]
    counts the calls that received one."""
    from kge_b200 import engine

    repl = {"train_1vsall_forward": _train_1vsall_forward, "train_1vsall_backward": _train_1vsall_backward,
            "score_1vsN_loss_csr": _score_1vsN_loss_csr,
            "score_1vsN_loss_csr_backward": _score_1vsN_loss_csr_backward}
    with engine_stub.installed():
        saved = {k: getattr(engine, k) for k in repl}
        for k, v in repl.items():
            setattr(engine, k, v)
        try:
            yield
        finally:
            for k, v in saved.items():
                setattr(engine, k, v)


# ---- the reference job with the mirror's masks -------------------------------------------------------------------
class _Holder:
    key = None
    direction = 0
    count = {"ent": 0, "rel": 0}

    def begin(self, direction):
        self.direction = direction
        self.count = {"ent": 0, "rel": 0}


class MirrorDropout(torch.nn.Module):
    """Stands in for an embedder's torch.nn.Dropout: applies the mirror's mask of the stream that the current call
    has in the reference's order (score_sp: embed(s) 0, embed(p) 1, embed_all() 2; score_po: embed_all() 3, embed(o) 5,
    embed(p) 4) under the current sub-batch's key."""

    def __init__(self, p, holder, kind):
        super().__init__()
        self.p, self.holder, self.kind = p, holder, kind

    def forward(self, x):
        h = self.holder
        i = h.count[self.kind]
        h.count[self.kind] += 1
        if self.kind == "rel":
            stream = (SP_REL, PO_REL)[h.direction]
        else:
            stream = ((SP_ENT, SP_TABLE), (PO_TABLE, PO_ENT))[h.direction][i]
        table = stream in (SP_TABLE, PO_TABLE)
        k = h.key
        return apply(x, self.p, k.seed, k.call, stream, 0 if table else k.row_base)


def patch_reference_job(job, p_ent, p_rel):
    """Make an UNMODIFIED reference training job draw the mirror's masks with the plugin's keys: the embedders' dropout
    modules are replaced, score_sp / score_po mark the direction, and _process_subbatch sets the sub-batch's key."""
    from kge_b200 import engine
    from kge_b200.plugin.jobs import dropout_call

    holder = _Holder()
    model = job.model
    model.get_s_embedder().dropout = MirrorDropout(p_ent, holder, "ent")
    model.get_p_embedder().dropout = MirrorDropout(p_rel, holder, "rel")
    sp, po = model.score_sp, model.score_po

    def score_sp(*a, **kw):
        holder.begin(0)
        return sp(*a, **kw)

    def score_po(*a, **kw):
        holder.begin(1)
        return po(*a, **kw)

    model.score_sp, model.score_po = score_sp, score_po
    orig = job._process_subbatch
    state = {}

    def process(batch_index, batch, subbatch_slice, result):
        pos = (job.epoch, batch_index)
        ordinal = state["ordinal"] + 1 if state.get("pos") == pos else 0
        state.update(pos=pos, ordinal=ordinal)
        holder.key = engine.DropoutKey(p_ent, p_rel, torch.initial_seed(), dropout_call(job.epoch, batch_index, ordinal),
                                       subbatch_slice.start or 0)
        return orig(batch_index, batch, subbatch_slice, result)

    job._process_subbatch = process
    return job
