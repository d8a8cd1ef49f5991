"""TEST INFRASTRUCTURE: CPU mirror of KvsAll's s_o query type (relation prediction, score_so): the masked reference
expression of the loss under the dropout draws of streams 24-26 (include/b200kge.h), oracle-backed stand-ins of
engine.score_so_loss_csr / score_so_loss_csr_backward, and a patch that makes the REFERENCE job's score_so draw the
mirror's masks (an extension of tests/dropout_oracle.py, whose streams 0-5 it keeps)."""
from __future__ import annotations

import contextlib

import torch

import dropout_oracle as do
from oracle import kge_oracle as orc

SO_S, SO_O, SO_TABLE = 24, 25, 26


def so_scores(model, ent, rel, s, o, key=None):
    """score_so(s, o) [n, R] (kge_model.py:727-747), with the three s_o draws of `key` when given."""
    se, oe, r = ent[s.long()], ent[o.long()], rel
    if key is not None:
        se = do.apply(se, key.p_ent, key.seed, key.call, SO_S, key.row_base)
        oe = do.apply(oe, key.p_ent, key.seed, key.call, SO_O, key.row_base)
        r = do.apply(rel, key.p_rel, key.seed, key.call, SO_TABLE, 0)
    return orc.score_emb(model, se, r, oe, "s_o")


def csr_labels(offs, cols, n, m, dtype):
    """The dense [n, m] multi-hot labels of CSR rows (a repeated column counts as often as it appears)."""
    y = torch.zeros((n, m), dtype=dtype)
    counts = (offs[1:] - offs[:-1]).cpu()
    rows = torch.repeat_interleave(torch.arange(n), counts)
    y.index_put_((rows, cols.long().cpu()), torch.ones(len(rows), dtype=dtype), accumulate=True)
    return y


def loss_so(model, ent, rel, s, o, offs, cols, loss, offset, key=None):
    """Sum over rows of the s_o KvsAll loss (never smoothed, train_KvsAll.py:263)."""
    x = so_scores(model, ent, rel, s, o, key)
    y = csr_labels(offs, cols, x.shape[0], x.shape[1], x.dtype).to(x.device)
    return orc.bce_loss(x, y, offset) if loss == "bce" else orc.kl_loss(x, y)


# ---- engine stand-ins (CPU) ----------------------------------------------------------------------------------------
calls = {"so": 0, "so_dropout": 0}


def _score_so_loss_csr(model, ent, rel, s, o, csr_offsets, csr_cols, loss="kl", offset=0.0, precision="auto",
                       return_rows=False, dropout=None):
    calls["so"] += 1
    calls["so_dropout"] += dropout is not None
    return loss_so(model, ent, rel, s, o, csr_offsets, csr_cols, loss, offset, dropout)


def _score_so_loss_csr_backward(model, ent, rel, s, o, csr_offsets, csr_cols, loss="kl", offset=0.0, batch_size=None,
                                dropout=None):
    calls["so"] += 1
    calls["so_dropout"] += dropout is not None
    bs = batch_size or s.numel()
    return do.grads(lambda e, r: loss_so(model, e, r, s, o, csr_offsets, csr_cols, loss, offset, dropout) / bs,
                    ent, rel)[1:]


@contextlib.contextmanager
def installed():
    """dropout_oracle.installed() plus the two s_o stand-ins; calls counts their calls."""
    from kge_b200 import engine

    repl = {"score_so_loss_csr": _score_so_loss_csr, "score_so_loss_csr_backward": _score_so_loss_csr_backward}
    with do.installed():
        saved = {k: getattr(engine, k) for k in repl}
        for k, v in repl.items():
            setattr(engine, k, v)
        try:
            yield calls
        finally:
            for k, v in saved.items():
                setattr(engine, k, v)


# ---- the reference job with the mirror's masks -------------------------------------------------------------------
SO_DIRECTION = 2


class MirrorDropoutSo(do.MirrorDropout):
    """dropout_oracle.MirrorDropout plus score_so's draws: embed(s) 24, embed(o) 25, embed_all() of the relations 26."""

    def forward(self, x):
        h = self.holder
        if h.direction != SO_DIRECTION:
            return super().forward(x)
        i = h.count[self.kind]
        h.count[self.kind] += 1
        k = h.key
        if self.kind == "rel":
            return do.apply(x, self.p, k.seed, k.call, SO_TABLE, 0)
        return do.apply(x, self.p, k.seed, k.call, (SO_S, SO_O)[i], k.row_base)


def patch_reference_job(job, p_ent, p_rel):
    """dropout_oracle.patch_reference_job, with score_so drawing streams 24-26."""
    do.patch_reference_job(job, p_ent, p_rel)
    model = job.model
    holder = model.get_s_embedder().dropout.holder
    model.get_s_embedder().dropout = MirrorDropoutSo(p_ent, holder, "ent")
    model.get_p_embedder().dropout = MirrorDropoutSo(p_rel, holder, "rel")
    so = model.score_so

    def score_so(*a, **kw):
        holder.begin(SO_DIRECTION)
        return so(*a, **kw)

    model.score_so = score_so
    return job
