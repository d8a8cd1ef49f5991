"""LibKGE plugin: the reference's own model classes with the scoring path served by libb200kge.

Usage (unchanged LibKGE jobs, README.md:522-563 plugin mechanism):

    modules: [kge.job, kge.model, kge.model.embedder, kge_b200.plugin]
    model: b200_complex            # or b200_distmult / b200_simple / b200_cp / b200_rescal /
                                   #    b200_transe / b200_rotate

`b200_<model>.yaml` in this directory mirrors the reference's `<model>.yaml` (same embedder keys, so
`_entity_embedder._embeddings.weight` checkpoints load unchanged) and adds `precision`.
The classes subclass the reference's `KgeModel` / `RelationalScorer` (kge_model.py:122,354):

 * `score_emb(s_emb, p_emb, o_emb, combine)` (scorer level) → b200kge_score_spo / score_1vsN; this also
   serves `ReciprocalRelationsModel`, which calls the scorer directly
   (reciprocal_relations_model.py:76-124).
 * `score_spo / score_sp / score_po / score_sp_po` (model level) → index-level entry points that read
   the embedding tables in place (the LookupEmbedder gather is fused, no `embed_all()` table copy)
   whenever both embedders are plain LookupEmbedders with dropout inactive; otherwise the
   reference's embedders run and the scorer-level path takes over.
 * with embedding dropout active in training, the 1vsAll / KvsAll job plugins take the dropout entry points
   (`loss_1vsall` / `loss_kvsall*` with an engine.DropoutKey: masks drawn on the device with the distribution of the
   reference's draws), and so does the negative-sampling job plugin with `user.b200_ns_dropout: true`
   (`loss_negatives` / `score_negatives` with a key); the unmodified jobs' score_sp / score_po and score_sp_po keep the
   routes above.
 * extra fused methods `score_sp_loss / score_po_loss / rank_sp / rank_po` for job plugins.

CUDA only: CPU tensors raise (no fallback).  Backward (SURVEY 8f-1, "next") is provided by
recomputation through the reference's own dense expression inside a torch.autograd.Function.

This module needs the reference package `kge` to be importable; kge_b200's standalone mirror
(kge_b200.model) does not.
"""
from __future__ import annotations

import torch

from kge.model import ComplEx, CP, DistMult, Rescal, RotatE, SimplE, TransE
from kge.model.complex import ComplExScorer
from kge.model.cp import CPScorer
from kge.model.distmult import DistMultScorer
from kge.model.embedder.lookup_embedder import LookupEmbedder
from kge.model.rescal import RescalScorer
from kge.model.rotate import RotatEScorer
from kge.model.simple import SimplEScorer
from kge.model.transe import TransEScorer

from .. import engine
from .._lib import NS_P_MAX_RELATIONS


class _ScoreEmbFn(torch.autograd.Function):
    """Forward: sm_90a kernels.  Backward: recompute with the reference's dense expression."""

    @staticmethod
    def forward(ctx, scorer, ref_score_emb, combine, s_emb, p_emb, o_emb):
        ctx.ref, ctx.combine = ref_score_emb, combine
        ctx.save_for_backward(s_emb, p_emb, o_emb)
        return scorer._b200_forward(s_emb.detach(), p_emb.detach(), o_emb.detach(), combine)

    @staticmethod
    def backward(ctx, grad_out):
        s, p, o = (t.detach().requires_grad_(True) for t in ctx.saved_tensors)
        with torch.enable_grad():
            out = ctx.ref(s, p, o, ctx.combine)
            gs, gp, go = torch.autograd.grad(out, (s, p, o), grad_out.reshape(out.shape), allow_unused=True)
        return None, None, None, gs, gp, go


class _B200ScorerMixin:
    _b200_name = None

    def _b200_l_norm(self):
        return float(getattr(self, "_norm", 1.0))

    def _b200_precision(self):
        try:
            return self.get_option("precision")
        except Exception:
            return "auto"

    def _b200_forward(self, s_emb, p_emb, o_emb, combine):
        name, ln, prec = self._b200_name, self._b200_l_norm(), self._b200_precision()
        n = p_emb.size(0)
        if combine == "spo":
            return engine.score_spo(name, s_emb, p_emb, o_emb, l_norm=ln).view(n, -1)
        if combine == "sp_":
            return engine.score_1vsN(name, "sp_", s_emb, p_emb, o_emb, l_norm=ln, precision=prec)
        if combine == "_po":
            return engine.score_1vsN(name, "_po", o_emb, p_emb, s_emb, l_norm=ln, precision=prec)
        raise ValueError(combine)

    def score_emb(self, s_emb, p_emb, o_emb, combine: str):
        if combine not in ("spo", "sp_", "_po"):
            # "s_o" is outside the fused scope: generic expansion of the base class, which lands
            # in this class again with combine="spo" (kge_model.py:200-209)
            return super().score_emb(s_emb, p_emb, o_emb, combine)
        ref = super().score_emb
        needs_grad = torch.is_grad_enabled() and any(t.requires_grad for t in (s_emb, p_emb, o_emb))
        if needs_grad:
            return _ScoreEmbFn.apply(self, ref, combine, s_emb, p_emb, o_emb)
        return self._b200_forward(s_emb, p_emb, o_emb, combine)


def _scorer(name, base):
    return type(f"B200{base.__name__}", (_B200ScorerMixin, base), {"_b200_name": name})


class _TableScoreFn(torch.autograd.Function):
    """Index-level scoring that reads the embedding tables in place.  Forward: sm_90a kernels (gather fused,
    no `embed_all()` copy).  Backward: `model._b200_score_backward` (gradient kernels where validated, else
    recomputation through the reference's dense expression)."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, kind, a, p, b):
        ctx.model, ctx.kind = model, kind
        ctx.save_for_backward(ent_w, rel_w, a, p, b if b is not None else torch.empty(0, device=ent_w.device))
        ctx.has_b = b is not None
        return model._b200_score_forward(ent_w.detach(), rel_w.detach(), kind, a, p, b)

    @staticmethod
    def backward(ctx, grad_out):
        ent_w, rel_w, a, p, b = ctx.saved_tensors
        d_ent, d_rel = ctx.model._b200_score_backward(ent_w, rel_w, ctx.kind, a, p, b if ctx.has_b else None,
                                                      grad_out)
        return d_ent, d_rel, None, None, None, None, None


class _Loss1vsAllFn(torch.autograd.Function):
    """Fused 1vsAll step: (loss(score_sp, o) + loss(score_po, s)) / n as ONE launch sequence.  With a dropout key
    (engine.DropoutKey) the step applies embedding dropout and the backward regenerates the same masks from the key."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, triples, loss, offset, dropout=None, reciprocal=None):
        ctx.model, ctx.loss, ctx.offset, ctx.dropout, ctx.reciprocal = model, loss, offset, dropout, reciprocal
        ctx.save_for_backward(ent_w, rel_w, triples)
        ln, prec = model._b200_args()
        if reciprocal is not None:
            return engine.train_1vsall_reciprocal_forward(model._b200_name, ent_w.detach(), rel_w.detach(), triples,
                                                          reciprocal, loss, offset, ln, prec, dropout=dropout)
        kw = {} if dropout is None else {"dropout": dropout}
        return engine.train_1vsall_forward(model._b200_name, ent_w.detach(), rel_w.detach(), triples, loss, offset,
                                           ln, prec, **kw)

    @staticmethod
    def backward(ctx, g):
        ent_w, rel_w, triples = ctx.saved_tensors
        if ctx.reciprocal is not None:
            d_ent, d_rel = engine.train_1vsall_reciprocal_backward(
                ctx.model._b200_name, ent_w.detach(), rel_w.detach(), triples, ctx.reciprocal, ctx.loss, ctx.offset,
                ctx.model._b200_args()[0], dropout=ctx.dropout)
        else:
            d_ent, d_rel = ctx.model._b200_loss_1vsall_backward(ent_w, rel_w, triples, ctx.loss, ctx.offset, ctx.dropout)
        return d_ent * g, d_rel * g, None, None, None, None, None, None


def _penalty_torch(emb, w, regularize, rw, p, weighted, indexes):
    """LookupEmbedder.penalty's expression (lookup_embedder.py:123-177) on a weight tensor — the differentiable
    form behind _PenaltyFn.backward."""
    if not weighted:
        par = emb._abs_complex(w) if (regularize == "n3" and emb.space == "complex") else w
        return (rw / p * par.norm(p=p) ** p).sum()
    uniq, counts = torch.unique(indexes, return_counts=True)
    par = w[uniq.long()]
    if regularize == "n3" and emb.space == "complex":
        par = emb._abs_complex(par)
    if (p % 2 == 1) and regularize != "n3":
        par = torch.abs(par)
    return (rw / p * (par ** p * counts.float().view(-1, 1))).sum() / len(indexes)


def _sparse_scaled(d, g):
    """d * g for a dense or a coalesced sparse COO gradient (only the values are scaled)."""
    if not d.is_sparse:
        return d * g
    return torch.sparse_coo_tensor(d._indices(), d._values() * g, d.shape, is_coalesced=True)


class _PenaltyFn(torch.autograd.Function):
    """Forward: the Lp / N3 row kernel (b200kge_lookup_penalty).  Backward: autograd of the reference expression; for
    a `sparse: True` embedder row-sparse over the rows the reference looks up: the unique indexes of the weighted
    penalty (self._embeddings(unique_indexes), lookup_embedder.py:155), every row of the unweighted one
    (self._embeddings_all(), :139)."""

    @staticmethod
    def forward(ctx, w, emb, regularize, rw, p, weighted, indexes):
        ctx.args = (emb, regularize, rw, p, weighted, indexes)
        ctx.save_for_backward(w)
        return engine.lookup_penalty(w.detach(), regularize, rw, float(p), weighted, indexes, emb.space)

    @staticmethod
    def backward(ctx, g):
        (w,) = ctx.saved_tensors
        wd = w.detach().requires_grad_(True)
        with torch.enable_grad():
            (gw,) = torch.autograd.grad(_penalty_torch(ctx.args[0], wd, *ctx.args[1:]), wd)
        emb, weighted, indexes = ctx.args[0], ctx.args[4], ctx.args[5]
        if emb.sparse:
            if weighted:
                rows = torch.unique(indexes).long()
                vals = gw[rows] * g
            else:
                rows = torch.arange(gw.shape[0], device=gw.device)
                vals = gw * g
            return (torch.sparse_coo_tensor(rows[None, :], vals, gw.shape, is_coalesced=True),
                    None, None, None, None, None, None)
        return gw * g, None, None, None, None, None, None


def _install_embedder_kernels(emb):
    """Serve a plain LookupEmbedder's penalty() and _normalize_embeddings() (lookup_embedder.py:64-69,122-177) from
    the row kernels of libb200kge when its table lives on a CUDA device.  Patched on the INSTANCE: class, parameter
    names and checkpoints stay the reference's; the post-batch normalisation hooks (prepare_job, :71-80) pick the
    patched method up through `self`."""
    if type(emb) is not LookupEmbedder or getattr(emb, "_b200_patched", False):
        return
    cls = type(emb)

    def penalty(**kwargs):
        w = emb._embeddings.weight
        # the reference's penalty reads _embeddings directly, so dropout never enters it (lookup_embedder.py:139,153)
        if not w.is_cuda or emb.regularize not in ("lp", "n3") or emb.get_option("regularize_weight") == 0.0:
            return cls.penalty(emb, **kwargs)
        if emb.regularize == "n3":
            p = 3
        else:
            p = emb.get_option("regularize_args.p") if emb.has_option("regularize_args.p") else 2
        weighted = bool(emb.get_option("regularize_args.weighted"))
        indexes = kwargs.get("indexes") if weighted else None
        rw = emb._get_regularize_weight()
        if torch.is_grad_enabled() and w.requires_grad:
            val = _PenaltyFn.apply(w, emb, emb.regularize, rw, p, weighted, indexes)
        else:
            val = engine.lookup_penalty(w.detach(), emb.regularize, rw, float(p), weighted, indexes, emb.space)
        return super(cls, emb).penalty(**kwargs) + [(f"{emb.configuration_key}.L{p}_penalty", val)]

    def _normalize_embeddings():
        w = emb._embeddings.weight
        if emb.normalize_p > 0 and w.is_cuda and w.is_contiguous():
            with torch.no_grad():
                engine.normalize_rows_(w.data, float(emb.normalize_p))
        else:
            cls._normalize_embeddings(emb)

    emb.penalty = penalty
    emb._normalize_embeddings = _normalize_embeddings
    emb._b200_patched = True


class _KvsAllLossFn(torch.autograd.Function):
    """KvsAll loss of one query type with CSR labels / batch_size: forward = fused score + loss with the CSR consumed in
    the epilogue; backward = the gradient kernels (b200kge_score_1vsN_loss_csr_backward; for combine "s_o" the pairs
    (a, p) = (s, o) against the relation table, b200kge_score_so_loss_csr and its backward).  With a dropout key both run
    the dropout forms (b200kge_score_1vsN_loss_csr_dropout, the backward with its dropout key) under the same masks."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, combine, a, p, offs, cols, loss, offset, smoothing, batch_size, dropout=None,
                dropout_streams=None):
        ctx.args = (model, combine, loss, offset, smoothing, batch_size, dropout, dropout_streams)
        ctx.save_for_backward(ent_w, rel_w, a, p, offs, cols)
        ln, prec = model._b200_args()
        kw = {} if dropout is None else {"dropout": dropout}
        if combine == "s_o":      # a = s, p = o; the relation targets are never smoothed
            return engine.score_so_loss_csr(model._b200_name, ent_w.detach(), rel_w.detach(), a, p, offs, cols, loss,
                                            offset, prec, **kw) / batch_size
        if dropout_streams is not None:
            kw["dropout_streams"] = dropout_streams
        return engine.score_1vsN_loss_csr(model._b200_name, combine, ent_w.detach(), rel_w.detach(), ent_w.detach(), offs,
                                          cols, a, p, loss, offset, smoothing, ln, prec, **kw) / batch_size

    @staticmethod
    def backward(ctx, g):
        ent_w, rel_w, a, p, offs, cols = ctx.saved_tensors
        model, combine, loss, offset, smoothing, batch_size, dropout, dropout_streams = ctx.args
        kw = {} if dropout is None else {"dropout": dropout}
        if combine == "s_o":
            d_ent, d_rel = engine.score_so_loss_csr_backward(model._b200_name, ent_w.detach(), rel_w.detach(), a, p, offs,
                                                             cols, loss, offset, batch_size, **kw)
            return (d_ent * g, d_rel * g) + (None,) * 12
        if dropout_streams is not None:
            kw["dropout_streams"] = dropout_streams
        if model._b200_name in ("transe", "rotate"):
            kw["l_norm"] = model._b200_args()[0]
        d_ent, d_rel = engine.score_1vsN_loss_csr_backward(model._b200_name, combine, ent_w.detach(), rel_w.detach(), a, p,
                                                           offs, cols, loss, offset, smoothing, batch_size, **kw)
        return (d_ent * g, d_rel * g) + (None,) * 12


class _NsSlotLossFn(torch.autograd.Function):
    """One slot of a negative-sampling batch: forward = fused gather+score [n, 1+K] and the loss kernel; backward = the
    fused NS gradient kernel (b200kge_ns_backward: per-row fold, per-column recompute, scatter).  BCE runs the dense-loss
    kernel and the kernel's own BCE gradient; every other loss runs the row-loss kernel (b200kge_ns_loss), which also
    writes G = dL/dscores, and the backward reads G (b200kge_ns_backward with grad_scores).  With a dropout key (engine.DropoutKey)
    the forward scores the masked block (b200kge_ns_score_dropout, draws of `implementation`), every loss BCE included
    runs the row-loss kernel, and the backward regenerates the same masks from the key (b200kge_ns_backward with the
    key).  When an embedder has `sparse: True` the backward is b200kge_ns_backward_sparse instead: that table's
    gradient is row-sparse over the rows the reference looks up (every entity row for `implementation` "all")."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, triples, negatives, slot, offset, batch_size, loss="bce", temperature=1.0,
                dropout=None, implementation="batch"):
        ctx.args = (model, slot, offset, batch_size, loss, dropout, implementation)
        ln = model._b200_args()[0]
        if dropout is not None:
            scores = engine.ns_score(model._b200_name, ent_w.detach(), rel_w.detach(), triples, negatives, slot, True,
                                     ln, dropout=dropout, implementation=implementation)
            value, G = engine.ns_loss(scores, loss, offset, temperature, batch_size=batch_size, want_grad=True)
            ctx.save_for_backward(ent_w, rel_w, triples, negatives, G)
            return value
        scores = engine.ns_score(model._b200_name, ent_w.detach(), rel_w.detach(), triples, negatives, slot, True, ln)
        if loss == "bce":
            ctx.save_for_backward(ent_w, rel_w, triples, negatives)
            lab = torch.zeros(triples.shape[0], dtype=torch.int64, device=triples.device)
            return engine.loss_dense(scores, lab, "bce", offset) / batch_size
        value, G = engine.ns_loss(scores, loss, offset, temperature, batch_size=batch_size, want_grad=True)
        ctx.save_for_backward(ent_w, rel_w, triples, negatives, G)
        return value

    @staticmethod
    def backward(ctx, g):
        model, slot, offset, batch_size, loss, dropout, implementation = ctx.args
        ent_w, rel_w, triples, negatives = ctx.saved_tensors[:4]
        sparse = model.b200_sparse_grads()
        if any(sparse):
            kw = {"sparse": sparse, "implementation": implementation}
            if dropout is not None or loss != "bce":
                kw["grad_scores"] = ctx.saved_tensors[4]
            if dropout is not None:
                kw["dropout"] = dropout
            d_ent, d_rel = engine.ns_backward_sparse(model._b200_name, ent_w.detach(), rel_w.detach(), triples, slot,
                                                     negatives, offset, model._b200_args()[0], batch_size, **kw)
            return (_sparse_scaled(d_ent, g), _sparse_scaled(d_rel, g)) + (None,) * 10
        if dropout is not None:
            kw = {"grad_scores": {slot: ctx.saved_tensors[4]}, "dropout": dropout, "implementation": implementation}
        else:
            kw = {} if loss == "bce" else {"grad_scores": {slot: ctx.saved_tensors[4]}}
        d_ent, d_rel = engine.ns_backward(model._b200_name, ent_w.detach(), rel_w.detach(), triples, {slot: negatives},
                                          offset, model._b200_args()[0], batch_size, **kw)
        return (d_ent * g, d_rel * g) + (None,) * 10


class _NsPSlotLossFn(torch.autograd.Function):
    """The P slot of a negative-sampling batch (relation negatives): forward = the fused gather+score [n, 1+K]
    (b200kge_ns_score, slot 1) and the row-loss kernel, which writes G = dL/dscores for every loss, BCE included;
    backward = b200kge_ns_p_backward, which sums G into one coefficient per (row, relation) before any table gradient is
    formed.  A `sparse: True` embedder gets its gradient row-sparse over the rows score_so looks up (every relation row
    for `implementation` "all")."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, triples, negatives, offset, batch_size, loss, temperature, implementation):
        ctx.args = (model, implementation)
        scores = engine.ns_score(model._b200_name, ent_w.detach(), rel_w.detach(), triples, negatives, 1, True,
                                 model._b200_args()[0])
        value, G = engine.ns_loss(scores, loss, offset, temperature, batch_size=batch_size, want_grad=True)
        ctx.save_for_backward(ent_w, rel_w, triples, negatives, G)
        return value

    @staticmethod
    def backward(ctx, g):
        model, implementation = ctx.args
        ent_w, rel_w, triples, negatives, G = ctx.saved_tensors
        d_ent, d_rel = engine.ns_p_backward(model._b200_name, ent_w.detach(), rel_w.detach(), triples, negatives, G,
                                            model._b200_args()[0], implementation, sparse=model.b200_sparse_grads())
        return (_sparse_scaled(d_ent, g), _sparse_scaled(d_rel, g)) + (None,) * 8


class _NsSharedLossFn(torch.autograd.Function):
    """One S / O slot of a negative-sampling batch under shared sampling (`negative_sampling.shared: True`): forward =
    b200kge_ns_shared_score (the fixed pair of every row scored against the U' shared rows, assembled into the
    [n, 1+K] block in the reference's column order) and the row-loss kernel, which writes G = dL/dscores for every
    loss; backward = b200kge_ns_shared_backward, which sums G per shared id before any table gradient is formed.  The
    scores against the shared rows are kept for TransE l_norm 2, whose backward divides by them.  A `sparse: True`
    embedder gets its gradient row-sparse over the rows the reference looks up under `implementation`."""

    @staticmethod
    def forward(ctx, ent_w, rel_w, model, triples, slot, unique, repeat, drop, K, offset, batch_size, loss, temperature,
                implementation):
        ln, prec = model._b200_args()
        l2 = model._b200_name == "transe" and ln == 2.0
        out = engine.ns_shared_score(model._b200_name, ent_w.detach(), rel_w.detach(), triples, slot, unique, repeat,
                                     drop, K, ln, prec, implementation, want_z=l2)
        scores, z = out if l2 else (out, None)
        value, G = engine.ns_loss(scores, loss, offset, temperature, batch_size=batch_size, want_grad=True)
        ctx.args = (model, slot, K, implementation)
        ctx.save_for_backward(ent_w, rel_w, triples, unique, repeat, drop, G, z)
        return value

    @staticmethod
    def backward(ctx, g):
        model, slot, K, implementation = ctx.args
        ent_w, rel_w, triples, unique, repeat, drop, G, z = ctx.saved_tensors
        d_ent, d_rel = engine.ns_shared_backward(model._b200_name, ent_w.detach(), rel_w.detach(), triples, slot, unique,
                                                 repeat, drop, K, G, z, model._b200_args()[0], implementation,
                                                 sparse=model.b200_sparse_grads())
        return (_sparse_scaled(d_ent, g), _sparse_scaled(d_rel, g)) + (None,) * 12


class _B200ModelMixin:
    """Index-level overrides (kge_model.py:663-789): read the tables in place when possible."""

    _b200_name = None
    _b200_scorer_cls = None
    #: "native": gradient kernels of libb200kge where they exist (fused 1vsAll step of the dot family with bce / kl:
    #: recompute, G planes, two split-K tensor-core GEMMs, unfold — validated against the reference's gradients);
    #: "reference": recompute through the reference's dense torch expression (autograd) — also what every other
    #: combination falls back to
    b200_backward = "native"

    def __init__(self, config, dataset, configuration_key=None, init_for_load_only=False):
        super().__init__(config=config, dataset=dataset, configuration_key=configuration_key,
                         init_for_load_only=init_for_load_only)
        # swap the reference scorer for ours (same configuration key, same options)
        self._scorer = self._b200_scorer_cls(config, dataset, self.configuration_key)
        # penalties and row normalisation of plain LookupEmbedders through the row kernels (SURVEY 8f-3)
        for emb in {id(e): e for e in (self.get_s_embedder(), self.get_p_embedder(), self.get_o_embedder())}.values():
            _install_embedder_kernels(emb)

    # -- helpers
    def b200_fusable(self):
        """True if the tables can be read in place: plain LookupEmbedders, one entity table, dropout inactive."""
        key = self.training
        cached = self.__dict__.get("_b200_fusable_cache")
        if cached is not None and cached[0] == key:          # embedder types / dropout rates are fixed after creation
            return cached[1]
        ok = self._b200_fusable_now()
        self.__dict__["_b200_fusable_cache"] = (key, ok)
        return ok

    def _b200_fusable_now(self):
        es, ep, eo = self.get_s_embedder(), self.get_p_embedder(), self.get_o_embedder()
        for e in (es, ep, eo):
            if type(e) is not LookupEmbedder:
                return False
            if e.dropout.p > 0 and e.training:
                return False
        return es is eo

    def b200_dropout_rates(self):
        """(p_ent, p_rel) when embedding dropout is active (training mode, a rate > 0) on plain LookupEmbedders that
        share one entity table — the case the dropout entry points of the 1vsAll / KvsAll steps serve — else None.
        Independent of b200_fusable(), which stays False while dropout is active."""
        es, ep, eo = self.get_s_embedder(), self.get_p_embedder(), self.get_o_embedder()
        if es is not eo or type(es) is not LookupEmbedder or type(ep) is not LookupEmbedder:
            return None
        rates = tuple(float(e.dropout.p) if e.training else 0.0 for e in (es, ep))
        return rates if max(rates) > 0 else None

    def b200_csr_labels_ok(self, label_smoothing):
        """The CSR-label loss takes label smoothing for the dot family (Q . colsum(T)) and for TransE / RotatE (the row
        score sums of the CUDA-core scoring pass), every norm."""
        return label_smoothing == 0.0 or self._b200_name in ("complex", "distmult", "simple", "cp", "rescal", "transe",
                                                             "rotate")

    def _b200_weights(self):
        return self.get_s_embedder()._embeddings.weight, self.get_p_embedder()._embeddings.weight

    def _b200_tables(self):
        e, r = self._b200_weights()
        return e.detach(), r.detach()

    def _b200_args(self):
        sc = self._scorer
        return sc._b200_l_norm(), sc._b200_precision()

    def _b200_needs_grad(self):
        e, r = self._b200_weights()
        return torch.is_grad_enabled() and (e.requires_grad or r.requires_grad)

    def _b200_score_forward(self, ent, rel, kind, a, p, b):
        ln, prec = self._b200_args()
        name = self._b200_name
        if kind == "spo":
            return engine.score_spo(name, ent, rel, ent, a, p, b, ln).view(-1)
        if kind == "sp_":
            return engine.score_1vsN(name, "sp_", ent, rel, ent, a, p, b, ln, prec)
        if kind == "_po":
            return engine.score_1vsN(name, "_po", ent, rel, ent, a, p, b, ln, prec)
        if kind == "sp_po":   # a = [s | o] stacked
            n = p.numel()
            return engine.score_sp_po(name, ent, rel, a[:n], p, a[n:], b, ln, prec)
        raise ValueError(kind)

    def _b200_ref_scores(self, ent, rel, kind, a, p, b):
        """The reference's dense expression on gathered rows (for the recompute backward)."""
        ref = super(_B200ScorerMixin, self._scorer).score_emb
        if kind == "spo":
            return ref(ent[a], rel[p], ent[b], "spo").view(-1)
        cand = ent if b is None else ent[b]
        if kind == "sp_":
            return ref(ent[a], rel[p], cand, "sp_")
        if kind == "_po":
            return ref(cand, rel[p], ent[a], "_po")
        n = p.numel()
        return torch.cat((ref(ent[a[:n]], rel[p], cand, "sp_"), ref(cand, rel[p], ent[a[n:]], "_po")), dim=1)

    def _b200_native_family(self):
        """Models / norms whose 1-vs-N gradients the library computes itself."""
        name, ln = self._b200_name, self._b200_args()[0]
        return (name in ("complex", "distmult", "simple", "cp", "rescal")
                or (name == "transe" and ln in (1.0, 2.0)) or (name == "rotate" and ln == 1.0))

    def _b200_score_backward(self, ent_w, rel_w, kind, a, p, b, grad_out):
        name = self._b200_name
        if self.b200_backward == "native" and b is None and kind in ("sp_", "_po", "sp_po") and self._b200_native_family():
            # dense [n, E] (or [n, 2E]) scores over the whole table: tensor-core gradient GEMMs (dot family) or the
            # row-gradient passes (TransE L1 / L2, RotatE L1) + unfold
            E_ = ent_w.shape[0]
            ln = self._b200_args()[0]
            if kind != "sp_po":
                return engine.score_1vsN_backward(name, kind, ent_w.detach(), rel_w.detach(), a, p, grad_out, ln)
            n = p.numel()
            de1, dr1 = engine.score_1vsN_backward(name, "sp_", ent_w.detach(), rel_w.detach(), a[:n], p, grad_out[:, :E_], ln)
            de2, dr2 = engine.score_1vsN_backward(name, "_po", ent_w.detach(), rel_w.detach(), a[n:], p, grad_out[:, E_:], ln)
            return de1 + de2, dr1 + dr2
        e, r = ent_w.detach().requires_grad_(True), rel_w.detach().requires_grad_(True)
        with torch.enable_grad():
            out = self._b200_ref_scores(e, r, kind, a, p, b)
            return torch.autograd.grad(out, (e, r), grad_out.reshape(out.shape), allow_unused=False)

    def b200_1vsall_native_backward_ok(self):
        return self.b200_backward == "native" and self._b200_native_family()

    def _b200_loss_1vsall_backward(self, ent_w, rel_w, triples, loss, offset, dropout=None):
        name = self._b200_name
        ln = self._b200_args()[0]
        if dropout is not None:       # no recompute form: the engine refuses what its kernels do not cover
            return engine.train_1vsall_backward(name, ent_w.detach(), rel_w.detach(), triples, loss, offset, ln,
                                                dropout=dropout)
        if self.b200_1vsall_native_backward_ok():
            return engine.train_1vsall_backward(name, ent_w.detach(), rel_w.detach(), triples, loss, offset, ln)
        e, r = ent_w.detach().requires_grad_(True), rel_w.detach().requires_grad_(True)
        n = triples.shape[0]
        s, p, o = triples[:, 0], triples[:, 1], triples[:, 2]
        with torch.enable_grad():
            total = 0.0
            for kind, a, lab in (("sp_", s, o), ("_po", o, s)):
                x = self._b200_ref_scores(e, r, kind, a, p, None)
                if loss == "bce":
                    y = torch.zeros_like(x)
                    y[torch.arange(n, device=x.device), lab] = 1.0
                    total = total + torch.nn.functional.binary_cross_entropy_with_logits(x + offset, y, reduction="sum")
                else:
                    total = total + torch.nn.functional.cross_entropy(x, lab, reduction="sum")
            return torch.autograd.grad(total / n, (e, r))

    def _b200_call(self, kind, a, p, b):
        ent_w, rel_w = self._b200_weights()
        if self._b200_needs_grad():
            return _TableScoreFn.apply(ent_w, rel_w, self, kind, a, p, b)
        return self._b200_score_forward(ent_w.detach(), rel_w.detach(), kind, a, p, b)

    def score_spo(self, s, p, o, direction=None):
        if not self.b200_fusable():
            return super().score_spo(s, p, o, direction)
        return self._b200_call("spo", s, p, o)

    def score_sp(self, s, p, o=None):
        if not self.b200_fusable():
            return super().score_sp(s, p, o)
        return self._b200_call("sp_", s, p, o)

    def score_po(self, p, o, s=None):
        if not self.b200_fusable():
            return super().score_po(p, o, s)
        return self._b200_call("_po", o, p, s)

    def score_sp_po(self, s, p, o, entity_subset=None):
        if not self.b200_fusable():
            return super().score_sp_po(s, p, o, entity_subset)
        return self._b200_call("sp_po", torch.cat((s.reshape(-1), o.reshape(-1))), p, entity_subset)

    # -- fused forms for the job plugins (kge_b200/plugin/jobs.py): scores never reach HBM
    def loss_1vsall(self, triples, loss="bce", offset=0.0, need_grad=None, dropout=None, reciprocal=None):
        """(loss(score_sp, o) + loss(score_po, s)) / n for a [n,3] batch (train_1vsAll.py:48-82); `dropout` (an
        engine.DropoutKey) applies embedding dropout with the masks of that key.  `reciprocal` = R when this model is
        the base model of a ReciprocalRelationsModel (2R relation rows): score_po is then the sp_ query (o, p + R)
        (reciprocal_relations_model.py:85-92).  The reciprocal step has the native backward only."""
        ent_w, rel_w = self._b200_weights()
        if need_grad is None:
            need_grad = self._b200_needs_grad()
        if reciprocal is not None:
            if need_grad and self._b200_needs_grad():
                return _Loss1vsAllFn.apply(ent_w, rel_w, self, triples, loss, offset, dropout, int(reciprocal))
            ln, prec = self._b200_args()
            return engine.train_1vsall_reciprocal_forward(self._b200_name, ent_w.detach(), rel_w.detach(), triples,
                                                          int(reciprocal), loss, offset, ln, prec, dropout=dropout)
        if need_grad and self._b200_needs_grad():
            return _Loss1vsAllFn.apply(ent_w, rel_w, self, triples, loss, offset, dropout)
        if dropout is not None:
            ln, prec = self._b200_args()
            return engine.train_1vsall_forward(self._b200_name, ent_w.detach(), rel_w.detach(), triples, loss, offset,
                                               ln, prec, dropout=dropout)
        return self._b200_prepared_step(ent_w, rel_w, triples.shape[0], loss, offset)(triples)

    def _b200_prepared_step(self, ent_w, rel_w, n, loss, offset):
        """forward only: a prepared step (table views, workspace, output scalar set up once per table storage)"""
        st = self.__dict__.get("_b200_step")
        if st is None or st.cfg != (loss, offset) or not st.matches(ent_w, rel_w, n):
            ln, prec = self._b200_args()
            st = engine.Step1vsAll(self._b200_name, ent_w.detach(), rel_w.detach(), max(n, 1024), loss, offset, ln, prec)
            st.cfg = (loss, offset)
            self.__dict__["_b200_step"] = st
        return st

    def loss_1vsall_host(self, triples_host, loss="bce", offset=0.0) -> float:
        """loss_1vsall for a HOST batch (contiguous int64 [n,3]) as a Python float, forward only: the copy to the
        device, the kernels and the read-back of the scalar are one library call (train_1vsAll.py:59-77)."""
        ent_w, rel_w = self._b200_weights()
        return self._b200_prepared_step(ent_w, rel_w, triples_host.shape[0], loss, offset).call_host(triples_host)

    def loss_kvsall(self, combine, a, p, csr_offsets, csr_cols, loss="kl", offset=0.0, label_smoothing=0.0,
                    dropout=None, dropout_streams=None):
        """Sum over rows of the KvsAll loss with CSR multi-hot labels (train_KvsAll.py:242-294); forward only.
        `dropout` (an engine.DropoutKey) applies embedding dropout with the masks of that key, drawn on the streams of
        query type `dropout_streams` (default: `combine`'s; a reciprocal-relations _po query is the sp_ fold of
        (o, p + R) on the _po streams).  combine "s_o": the pairs (a, p) = (s, o) against every relation (relation
        ids as labels, no smoothing; see b200_kvsall_so_ok)."""
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        kw = {} if dropout is None else {"dropout": dropout}
        if combine == "s_o":
            return engine.score_so_loss_csr(self._b200_name, ent, rel, a, p, csr_offsets, csr_cols, loss, offset, prec,
                                            **kw)
        if dropout is not None and dropout_streams is not None:
            kw["dropout_streams"] = dropout_streams
        return engine.score_1vsN_loss_csr(self._b200_name, combine, ent, rel, ent, csr_offsets, csr_cols, a, p,
                                          loss, offset, label_smoothing, ln, prec, **kw)

    def b200_kvsall_native_backward_ok(self, dropout=False):
        """The KvsAll gradient kernels cover the dot family, TransE with l_norm 1 or 2 and RotatE with l_norm 1.  The
        distance family's CSR-label backward recomputes the scores on the CUDA cores, where the unmodified step without
        dropout keeps its stored dense scores and runs the same row-gradient passes on dL/dscores: that step is faster
        (TransE L1 13.0 vs 14.9 ms, RotatE L1 20.8 vs 23.6 ms, scripts/kvsall_distance_train_bench.py).  So TransE and
        RotatE take the CSR-label backward under embedding dropout (`dropout`), where the unmodified step recomputes
        through the reference expression instead."""
        if self.b200_backward != "native" or not self._b200_native_family():
            return False
        return dropout or self._b200_name not in ("transe", "rotate")

    def b200_kvsall_so_ok(self):
        """The s_o query type has fused forward and gradient kernels for the dot family, at the precisions of the
        entity-ranking job (auto, fp32, f16x3), with the native backward.  TransE and RotatE have no s_o fold."""
        return (self.b200_backward == "native" and self._b200_name in ("complex", "distmult", "simple", "cp", "rescal")
                and self._b200_args()[1] in ("auto", "fp32", "f16x3"))

    def loss_kvsall_train(self, combine, a, p, csr_offsets, csr_cols, loss, offset, label_smoothing, batch_size,
                          dropout=None, dropout_streams=None):
        """loss_kvsall / batch_size as a differentiable scalar (train_KvsAll.py:286-294)."""
        ent_w, rel_w = self._b200_weights()
        return _KvsAllLossFn.apply(ent_w, rel_w, self, combine, a.long().contiguous(), p.long().contiguous(),
                                   csr_offsets, csr_cols, loss, float(offset), float(label_smoothing), int(batch_size),
                                   dropout, None if dropout is None else dropout_streams)

    def score_negatives(self, triples, negatives, slot, dropout=None, implementation="batch"):
        """[n, 1+K]: the positive triple's score in column 0, its K corrupted versions after it
        (train_negative_sampling.py:139-148 + sampler.py:263-344); forward only.  `dropout` (an engine.DropoutKey)
        applies the slot's embedding-dropout draws of `implementation` ("triple" | "batch" | "all")."""
        ent, rel = self._b200_tables()
        kw = {} if dropout is None else {"dropout": dropout, "implementation": implementation}
        return engine.ns_score(self._b200_name, ent, rel, triples, negatives, slot, True, self._b200_args()[0], **kw)

    def b200_ns_dropout_ok(self, slot):
        """The negative-sampling dropout kernels cover the S / O slots of the dot family, TransE (L1, L2) and RotatE
        (L1), with row widths the masks' four-element groups divide (D % 4 == 0, D % 8 == 0 for the models that split a
        row into halves).  Like b200_ns_native_backward_ok, it needs b200_backward = "native"."""
        if self.b200_backward != "native" or slot not in (0, 2):
            return False
        ln = self._b200_args()[0]
        if not {"transe": ln in (1.0, 2.0), "rotate": ln == 1.0}.get(self._b200_name, True):
            return False
        D = self._b200_weights()[0].shape[1]
        return D % (8 if self._b200_name in ("complex", "simple", "cp", "rotate") else 4) == 0

    def loss_dense(self, scores, labels, loss="bce", offset=0.0):
        return engine.loss_dense(scores, labels, loss, offset)

    def b200_sparse_grads(self):
        """(entities, relations): whether each table's embedder asks for row-sparse gradients (`lookup_embedder.sparse`,
        nn.Embedding(sparse=True), lookup_embedder.py:36,45)."""
        return bool(self.get_s_embedder().sparse), bool(self.get_p_embedder().sparse)

    def b200_ns_native_backward_ok(self, slot):
        """The fused NS gradient kernel covers the S / O slots of the dot family, TransE (L1, L2) and RotatE (L1)."""
        if self.b200_backward != "native" or slot not in (0, 2):
            return False
        ln = self._b200_args()[0]
        return {"transe": ln in (1.0, 2.0), "rotate": ln == 1.0}.get(self._b200_name, True)

    def loss_negatives(self, triples, negatives, slot, offset, batch_size, loss="bce", temperature=1.0, dropout=None,
                       implementation="batch"):
        """KgeLoss of one slot's [n, 1+K] block (positive first) / batch_size, differentiable through the gradient
        kernel (train_negative_sampling.py:139-164).  `loss` is a name of engine.ns_loss; `offset` its argument (the BCE
        offset, or the margin of margin_ranking), `temperature` that of bce_self_adversarial.  `dropout` (an
        engine.DropoutKey) applies the slot's embedding-dropout draws of `implementation` in forward and backward; "all"
        draws those of "batch".  With a `sparse: True` embedder `implementation` also picks the row set of the sparse
        gradients (see _NsSlotLossFn)."""
        ent_w, rel_w = self._b200_weights()
        return _NsSlotLossFn.apply(ent_w, rel_w, self, triples.long().contiguous(), negatives.long().contiguous(),
                                   int(slot), float(offset), int(batch_size), loss, float(temperature), dropout,
                                   implementation)

    def b200_ns_p_slot_ok(self):
        """The P-slot backward (b200kge_ns_p_backward) covers the dot family, TransE (L1, L2) and RotatE (L1) with at most
        NS_P_MAX_RELATIONS relations, and needs b200_backward = "native"."""
        return (self.b200_backward == "native" and self._b200_native_family()
                and self._b200_weights()[1].shape[0] <= NS_P_MAX_RELATIONS)

    def loss_negatives_p(self, triples, negatives, offset, batch_size, loss="bce", temperature=1.0,
                         implementation="batch"):
        """loss_negatives of the P slot: `negatives` [n, K] are relation ids, and the gradient comes from
        b200kge_ns_p_backward (see _NsPSlotLossFn; `implementation` only picks the row set of a sparse relation
        gradient).  No embedding dropout."""
        ent_w, rel_w = self._b200_weights()
        return _NsPSlotLossFn.apply(ent_w, rel_w, self, triples.long().contiguous(), negatives.long().contiguous(),
                                    float(offset), int(batch_size), loss, float(temperature), implementation)

    def b200_ns_shared_ok(self):
        """The shared-sampling kernels (b200kge_ns_shared_score / _backward) cover the dot family, TransE (L1, L2) and
        RotatE (L1) at the precisions auto, fp32 and f16x3 with a folded width of at most 1024, and need
        b200_backward = "native"."""
        ent_w = self._b200_weights()[0]
        width = ent_w.shape[1] // (2 if self._b200_name == "cp" else 1)
        return (self.b200_backward == "native" and self._b200_native_family() and width <= 1024
                and self._b200_args()[1] in ("auto", "fp32", "f16x3"))

    def loss_negatives_shared(self, triples, slot, unique, repeat, drop, num_samples, offset, batch_size, loss="bce",
                              temperature=1.0, implementation="batch"):
        """loss_negatives of one S / O slot under shared negative sampling: row i's K = num_samples negatives are the
        shared ids unique[u(i, c)] of engine.ns_shared_score (unique, repeat: the batch's _unique_samples and
        _repeat_indexes; drop: the sub-batch's rows of _drop_index, None for the naive type).  The gradient comes from
        b200kge_ns_shared_backward (see _NsSharedLossFn).  No embedding dropout."""
        ent_w, rel_w = self._b200_weights()
        return _NsSharedLossFn.apply(ent_w, rel_w, self, triples.long().contiguous(), int(slot), unique, repeat, drop,
                                     int(num_samples), float(offset), int(batch_size), loss, float(temperature),
                                     implementation)

    def loss_negatives_forward(self, scores, loss, arg=0.0, temperature=1.0):
        """Sum over rows of the KgeLoss of a scored [n, 1+K] block (positive first); forward only."""
        return engine.ns_loss(scores, loss, arg, temperature)[0]

    def score_sp_loss(self, s, p, labels, loss="bce", offset=0.0):
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        return engine.score_1vsN_loss(self._b200_name, "sp_", ent, rel, ent, labels, s, p, None, loss, offset, ln, prec)

    def score_po_loss(self, p, o, labels, loss="bce", offset=0.0):
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        return engine.score_1vsN_loss(self._b200_name, "_po", ent, rel, ent, labels, o, p, None, loss, offset, ln, prec)

    def rank_eval(self, s, p, o, true2n, F, T, rtol, atol, reciprocal=None, own_col=None):
        """Every ranking of an evaluation batch against the whole table in one call (engine.rank_sp_po_eval):
        F = (offsets, cols) the stacked-row CSR of the known answers, T the same for the test answers not in F, or None.
        `reciprocal` = R when this model is the base model of a ReciprocalRelationsModel.  own_col defaults to [o | s].
        Returns (rank, ties, own_score) with rank / ties [2 or 3, 2n]."""
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        if own_col is None:
            own_col = torch.cat((o.reshape(-1), s.reshape(-1)))
        return engine.rank_sp_po_eval(self._b200_name, ent, rel, s, p, o, true2n, own_col, F[0], F[1],
                                      None if T is None else T[0], None if T is None else T[1], rtol, atol, ln, prec,
                                      num_relations=int(reciprocal or 0))

    def rank_sp(self, s, p, true_scores, entity_subset=None, filter_labels=None, rtol=1e-4, atol=1e-5,
                rank=None, ties=None):
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        return engine.score_1vsN_rank(self._b200_name, "sp_", ent, rel, ent, true_scores, s, p, entity_subset,
                                      filter_labels, rtol, atol, ln, prec, rank, ties)

    def rank_po(self, p, o, true_scores, entity_subset=None, filter_labels=None, rtol=1e-4, atol=1e-5,
                rank=None, ties=None):
        ent, rel = self._b200_tables()
        ln, prec = self._b200_args()
        return engine.score_1vsN_rank(self._b200_name, "_po", ent, rel, ent, true_scores, o, p, entity_subset,
                                      filter_labels, rtol, atol, ln, prec, rank, ties)


def _model(cls_name, name, base_model, base_scorer):
    return type(cls_name, (_B200ModelMixin, base_model),
                {"_b200_name": name, "_b200_scorer_cls": _scorer(name, base_scorer)})


B200ComplEx = _model("B200ComplEx", "complex", ComplEx, ComplExScorer)
B200DistMult = _model("B200DistMult", "distmult", DistMult, DistMultScorer)
B200SimplE = _model("B200SimplE", "simple", SimplE, SimplEScorer)
B200CP = _model("B200CP", "cp", CP, CPScorer)
B200Rescal = _model("B200Rescal", "rescal", Rescal, RescalScorer)
B200TransE = _model("B200TransE", "transe", TransE, TransEScorer)
B200RotatE = _model("B200RotatE", "rotate", RotatE, RotatEScorer)

from .jobs import (B200EntityRankingJob, B200TrainingJob1vsAll, B200TrainingJobKvsAll,  # noqa: E402
                   B200TrainingJobNegativeSampling)

__all__ = ["B200ComplEx", "B200DistMult", "B200SimplE", "B200CP", "B200Rescal", "B200TransE", "B200RotatE",
           "B200TrainingJob1vsAll", "B200TrainingJobKvsAll", "B200TrainingJobNegativeSampling",
           "B200EntityRankingJob"]


def install_native_indexes(dataset, splits=("train", "valid", "test")):
    """Serve the dataset's `{split}_{sp|po|so}_to_{o|s|p}` indexes (kge/indexing.py:197-235) from
    kge_b200.indexing.KvsAllIndex — same attributes and accessors as the reference class (TrainingJobKvsAll's
    collate and EntityRankingJob's label lookup use it unchanged), built by the native sort/unique/lookup code
    instead of numpy + a numba dict.  Call once after the dataset is created."""
    from ..indexing import KvsAllIndex

    def make(split, key, cols, val, name):
        def fn(ds):
            if not ds._indexes.get(name):
                ds._indexes[name] = KvsAllIndex(ds.split(split), cols, val, torch.IntTensor)
            ds.config.log("{} distinct {} pairs in {}".format(len(ds._indexes[name]), key, split), prefix="  ")
            return ds._indexes.get(name)
        return fn

    for split in splits:
        for key, cols, val, v in (("sp", [0, 1], 2, "o"), ("po", [1, 2], 0, "s"), ("so", [0, 2], 1, "p")):
            name = f"{split}_{key}_to_{v}"
            dataset.index_functions[name] = make(split, key, cols, val, name)
            dataset._indexes.pop(name, None)
    return dataset
