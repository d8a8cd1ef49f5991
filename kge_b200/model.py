"""Host-side mirror of the reference's model interface for the scoring path.

Same names, argument meaning and error behaviour as LibKGE's

    KgeModel.score_spo / score_sp / score_po / score_so / score_sp_po    kge_model.py:663-789
    RelationalScorer.score_emb(s_emb, p_emb, o_emb, combine)             kge_model.py:151-213
    LookupEmbedder.embed / embed_all                                     lookup_embedder.py:96-112
    KgeLoss.create / __call__(scores, labels)                            loss.py:30-90,153,198
    BatchNegativeSample.score(model)                                     sampler.py:263-344
    EntityRankingJob._get_ranks_and_num_ties / _filter_and_rank / _get_ranks
                                                                         eval_entity_ranking.py:533-618

but standalone (the reference package is not required) and with every number produced by
libb200kge's sm_90a kernels.  The LibKGE plugin (kge_b200/plugin) wraps the same engine calls in
subclasses of the reference's own classes.  Forward only: backward is row (f)1 of SURVEY.md 8.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import engine

S, P, O = 0, 1, 2
SLOT_STR = ["s", "p", "o"]
MODEL_NAMES = ("complex", "distmult", "simple", "cp", "rescal", "transe", "rotate")


def relation_dim(model: str, dim: int) -> int:
    """cp.py:49-54, rotate.py:92-97 (D/2); rescal.py:78-95 (d*d); else D."""
    if model in ("cp", "rotate"):
        return dim // 2
    if model == "rescal":
        return dim * dim
    return dim


class LookupEmbedder(torch.nn.Module):
    """torch.nn.Embedding wrapper with the reference's parameter name (`_embeddings.weight`,
    lookup_embedder.py:44) so checkpoints load unchanged.  `embed`/`embed_all` exist for API
    parity; the scoring entry points read the table in place instead of calling them."""

    def __init__(self, vocab_size: int, dim: int, initialize: str = "normal_", sigma: float = 1.0):
        super().__init__()
        self.vocab_size, self.dim = vocab_size, dim
        self._embeddings = torch.nn.Embedding(vocab_size, dim)
        with torch.no_grad():
            if initialize == "normal_":
                self._embeddings.weight.normal_(0.0, sigma)
            elif initialize == "uniform_":
                self._embeddings.weight.uniform_(-sigma, sigma)
            else:
                raise ValueError(f"unknown initialize {initialize}")

    @property
    def weight(self) -> torch.Tensor:
        return self._embeddings.weight

    def embed(self, indexes: torch.Tensor) -> torch.Tensor:
        return self._embeddings(indexes.long())

    def embed_all(self) -> torch.Tensor:
        # the reference returns a fresh copy (lookup_embedder.py:107-112); a view is enough here
        return self._embeddings.weight


class RelationalScorer:
    """score_emb over already-gathered embeddings (what ReciprocalRelationsModel and user code
    call directly, reciprocal_relations_model.py:76-124)."""

    def __init__(self, model: str, l_norm: float = 1.0, precision: str = "auto"):
        if model not in MODEL_NAMES:
            raise ValueError(f"unknown model {model}")
        self.model, self.l_norm, self.precision = model, float(l_norm), precision

    def score_emb_spo(self, s_emb, p_emb, o_emb):
        return self.score_emb(s_emb, p_emb, o_emb, "spo")

    def score_emb(self, s_emb, p_emb, o_emb, combine: str):
        n = p_emb.size(0)
        if combine == "spo":
            assert s_emb.size(0) == n and o_emb.size(0) == n
            out = engine.score_spo(self.model, s_emb, p_emb, o_emb, l_norm=self.l_norm)
        elif combine == "sp_":
            assert s_emb.size(0) == n
            out = engine.score_1vsN(self.model, "sp_", s_emb, p_emb, o_emb, l_norm=self.l_norm,
                                    precision=self.precision)
        elif combine == "_po":
            assert o_emb.size(0) == n
            out = engine.score_1vsN(self.model, "_po", o_emb, p_emb, s_emb, l_norm=self.l_norm,
                                    precision=self.precision)
        elif combine == "s_o":
            n = s_emb.size(0)
            assert o_emb.size(0) == n
            m = p_emb.size(0)
            dev = s_emb.device
            rows = torch.arange(n, device=dev)
            tri = torch.stack([rows, torch.zeros_like(rows), rows], 1)
            neg = torch.arange(m, device=dev).unsqueeze(0).expand(n, m).contiguous()
            out = _ns_emb(self.model, s_emb, p_emb, o_emb, tri, neg, P, self.l_norm)
        else:
            raise ValueError('cannot handle combine="{}"'.format(combine))
        return out.view(n, -1)


def _ns_emb(model, s_emb, p_emb, o_emb, tri, neg, slot, l_norm):
    """score_so through the row-wise kernel with row divisors (relations as the open slot)."""
    import ctypes as C

    from . import _lib

    lib, k = _lib.load(), engine._Keep()
    rs = k.rows(s_emb, tri[:, S].contiguous())
    ro = k.rows(o_emb, tri[:, O].contiguous())
    # any valid per-row relation operand works for the (unused) positive relation rows
    rp = k.rows(p_emb, torch.zeros(tri.shape[0], dtype=torch.int64, device=tri.device))
    table = k.rows(p_emb)
    n, K = neg.shape
    out = torch.empty((n, K), dtype=torch.float32, device=s_emb.device)
    _lib.check(lib.b200kge_ns_score(_lib.MODELS[model], l_norm, C.byref(rs), C.byref(rp), C.byref(ro),
                                    C.byref(table), slot, neg.data_ptr(), n, K, 0, out.data_ptr(),
                                    out.stride(0), engine._stream(s_emb.device)))
    return out


class KgeModel(torch.nn.Module):
    """Index-level scoring façade (kge_model.py:354-789) over two LookupEmbedders and a scorer."""

    def __init__(self, model: str, num_entities: int, num_relations: int, dim: int,
                 l_norm: float = 1.0, sigma: float = 1.0, precision: str = "auto", seed: Optional[int] = None):
        super().__init__()
        if model not in MODEL_NAMES:
            raise ValueError(f"unknown model {model}")
        if model in ("complex", "simple", "cp", "rotate") and dim % 2 != 0:
            # simple.py:46-50, cp.py:44-48, rotate.py:87-91
            raise ValueError(f"{model} requires embeddings of even dimensionality (got {dim})")
        if seed is not None:
            torch.manual_seed(seed)
        self.model_name = model
        self._entity_embedder = LookupEmbedder(num_entities, dim, "normal_", sigma)
        if model == "rotate":  # phases ~ U(-pi, pi)   rotate.yaml:22-26
            self._relation_embedder = LookupEmbedder(num_relations, relation_dim(model, dim), "uniform_", math.pi)
        else:
            self._relation_embedder = LookupEmbedder(num_relations, relation_dim(model, dim), "normal_", sigma)
        self._scorer = RelationalScorer(model, l_norm, precision)

    # -- accessors (kge_model.py:651-661)
    def get_s_embedder(self): return self._entity_embedder
    def get_o_embedder(self): return self._entity_embedder
    def get_p_embedder(self): return self._relation_embedder
    def get_scorer(self): return self._scorer

    @property
    def _ent(self): return self._entity_embedder.weight.detach()
    @property
    def _rel(self): return self._relation_embedder.weight.detach()
    @property
    def l_norm(self): return self._scorer.l_norm
    @property
    def precision(self): return self._scorer.precision

    # -- the reference's five scoring methods
    def score_spo(self, s, p, o, direction=None) -> torch.Tensor:
        return engine.score_spo(self.model_name, self._ent, self._rel, self._ent, s, p, o, self.l_norm).view(-1)

    def score_sp(self, s, p, o=None) -> torch.Tensor:
        return engine.score_1vsN(self.model_name, "sp_", self._ent, self._rel, self._ent, s, p, o,
                                 self.l_norm, self.precision)

    def score_po(self, p, o, s=None) -> torch.Tensor:
        return engine.score_1vsN(self.model_name, "_po", self._ent, self._rel, self._ent, o, p, s,
                                 self.l_norm, self.precision)

    def score_so(self, s, o, p=None) -> torch.Tensor:
        dev = self._ent.device
        n = s.numel()
        tri = torch.stack([s.long(), torch.zeros_like(s.long()), o.long()], 1)
        cols = torch.arange(self._rel.shape[0], device=dev) if p is None else p.long()
        neg = cols.unsqueeze(0).expand(n, cols.numel()).contiguous()
        return engine.ns_score(self.model_name, self._ent, self._rel, tri, neg, P, False, self.l_norm)

    def score_sp_po(self, s, p, o, entity_subset=None) -> torch.Tensor:
        return engine.score_sp_po(self.model_name, self._ent, self._rel, s, p, o, entity_subset,
                                  self.l_norm, self.precision)

    # -- fused forms (scores never reach HBM); the LibKGE job plugins call these
    def score_sp_loss(self, s, p, labels, loss="bce", offset=0.0, o=None):
        return engine.score_1vsN_loss(self.model_name, "sp_", self._ent, self._rel, self._ent, labels, s, p, o,
                                      loss, offset, self.l_norm, self.precision)

    def score_po_loss(self, p, o, labels, loss="bce", offset=0.0, s=None):
        return engine.score_1vsN_loss(self.model_name, "_po", self._ent, self._rel, self._ent, labels, o, p, s,
                                      loss, offset, self.l_norm, self.precision)

    def rank_sp(self, s, p, true_scores, entity_subset=None, filter_labels=None, rtol=1e-4, atol=1e-5,
                rank=None, ties=None):
        return engine.score_1vsN_rank(self.model_name, "sp_", self._ent, self._rel, self._ent, true_scores, s, p,
                                      entity_subset, filter_labels, rtol, atol, self.l_norm, self.precision,
                                      rank, ties)

    def rank_po(self, p, o, true_scores, entity_subset=None, filter_labels=None, rtol=1e-4, atol=1e-5,
                rank=None, ties=None):
        return engine.score_1vsN_rank(self.model_name, "_po", self._ent, self._rel, self._ent, true_scores, o, p,
                                      entity_subset, filter_labels, rtol, atol, self.l_norm, self.precision,
                                      rank, ties)


class ReciprocalRelationsModel(KgeModel):
    """reciprocal_relations_model.py:16-124: a base model with 2R relation rows; row p + R is the reciprocal of
    relation p, and every query about subjects, (?, p, o), is answered as the object query (o, p + R, ?).  Only
    the index arithmetic lives here — all scoring goes through the same `sp_` entry points as the base model."""

    def __init__(self, model: str, num_entities: int, num_relations: int, dim: int, **kwargs):
        super().__init__(model, num_entities, 2 * num_relations, dim, **kwargs)
        self.num_relations = int(num_relations)

    def score_spo(self, s, p, o, direction=None) -> torch.Tensor:
        if direction == "o":
            return super().score_spo(s, p, o, "o")
        if direction == "s":
            return super().score_spo(o, p + self.num_relations, s, "o")
        raise Exception("The reciprocal relations model cannot compute undirected spo scores.")    # :79-82

    def score_po(self, p, o, s=None) -> torch.Tensor:
        return engine.score_1vsN(self.model_name, "sp_", self._ent, self._rel, self._ent, o, p + self.num_relations, s,
                                 self.l_norm, self.precision)

    def score_so(self, s, o, p=None):
        raise Exception("The reciprocal relations model cannot score relations.")                   # :94-95

    def score_sp_po(self, s, p, o, entity_subset=None) -> torch.Tensor:
        n = s.numel()
        m = self._ent.shape[0] if entity_subset is None else entity_subset.numel()
        out = torch.empty((n, 2 * m), dtype=torch.float32, device=self._ent.device)
        engine.score_1vsN(self.model_name, "sp_", self._ent, self._rel, self._ent, s, p, entity_subset, self.l_norm,
                          self.precision, out=out[:, :m])
        engine.score_1vsN(self.model_name, "sp_", self._ent, self._rel, self._ent, o, p + self.num_relations,
                          entity_subset, self.l_norm, self.precision, out=out[:, m:])
        return out

    def score_po_loss(self, p, o, labels, loss="bce", offset=0.0, s=None):
        return engine.score_1vsN_loss(self.model_name, "sp_", self._ent, self._rel, self._ent, labels, o,
                                      p + self.num_relations, s, loss, offset, self.l_norm, self.precision)

    def rank_po(self, p, o, true_scores, entity_subset=None, filter_labels=None, rtol=1e-4, atol=1e-5,
                rank=None, ties=None):
        return engine.score_1vsN_rank(self.model_name, "sp_", self._ent, self._rel, self._ent, true_scores, o,
                                      p + self.num_relations, entity_subset, filter_labels, rtol, atol, self.l_norm,
                                      self.precision, rank, ties)


class KgeLoss:
    """loss.py:20-274: `__call__(scores, labels)` with labels either a vector of positions or a label matrix; reduction
    is SUM (the caller divides by batch size).  bce / kl take any labels (the dense-loss kernel); bce_mean,
    bce_self_adversarial, margin_ranking, soft_margin and se take one positive per row — positions, or a 0/1 matrix with
    exactly one 1 per row such as the negative-sampling labels — on the row-loss kernel (margin_ranking pairs each
    row's positive with that row's other columns, the negative-sampling form of loss.py:240-252)."""

    ROW_WISE = ("bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se")

    def __init__(self, kind: str, offset: float = 0.0, temperature: float = 1.0):
        self.kind, self._offset, self._temperature = kind, offset, temperature

    @staticmethod
    def create(train_loss: str, loss_arg: float = float("nan")) -> "KgeLoss":
        """The losses of the 1vsAll / KvsAll steps (bce, kl)."""
        if train_loss == "bce":
            return KgeLoss("bce", 0.0 if math.isnan(loss_arg) else loss_arg)   # loss.py:46-52
        if train_loss == "kl":
            return KgeLoss("kl")
        raise ValueError("invalid value train.loss={}".format(train_loss))

    @staticmethod
    def create_negative_sampling(train_loss: str, loss_arg: float = float("nan"),
                                 temperature: float = 1.0) -> "KgeLoss":
        """Every loss a negative-sampling job accepts (loss.py:30-90 without ce), with the reference's loss_arg defaults:
        offset 0 for the BCE family, margin 1 for margin_ranking; `temperature` is
        user.bce_self_adversarial_temperature (loss.py:64-68)."""
        if train_loss in ("bce", "bce_mean", "bce_self_adversarial"):
            return KgeLoss(train_loss, 0.0 if math.isnan(loss_arg) else loss_arg, temperature)
        if train_loss == "margin_ranking":
            return KgeLoss("margin_ranking", 1.0 if math.isnan(loss_arg) else loss_arg)
        if train_loss in ("kl", "soft_margin", "se"):
            return KgeLoss(train_loss)
        raise ValueError("invalid value train.loss={}".format(train_loss))

    def __call__(self, scores, labels, **kwargs):
        if self.kind not in self.ROW_WISE:
            return engine.loss_dense(scores, labels, self.kind, self._offset)
        if labels.dim() == 2:
            # _labels_as_indexes (loss.py:119-136): exactly one 1 per row
            nz = labels.nonzero()
            if not nz[:, 0].equal(torch.arange(len(labels), device=labels.device)):
                raise ValueError("exactly one 1 per row required")
            labels = nz[:, 1]
        return engine.ns_loss(scores, self.kind, self._offset, self._temperature, label_idx=labels)[0]


class BatchNegativeSample:
    """sampler.py:212-356 (DefaultBatchNegativeSample): holds positive triples [n,3] and sampled
    indexes [n,K] for one slot; `score(model)` returns the [n,K] scores.  Both reference
    implementations (`triple`, `batch`) produce these same numbers; here the gather of the sampled
    rows is fused with the per-negative dot/distance."""

    def __init__(self, positive_triples: torch.Tensor, slot: int, samples: torch.Tensor):
        self.positive_triples, self.slot, self._samples = positive_triples, slot, samples
        self.num_samples = samples.shape[1]

    def samples(self, indexes=None):
        return self._samples if indexes is None else self._samples[indexes]

    def to(self, device):
        self.positive_triples = self.positive_triples.to(device)
        self._samples = self._samples.to(device)
        return self

    def score(self, model: KgeModel, indexes=None) -> torch.Tensor:
        neg = self.samples(indexes)
        tri = self.positive_triples[indexes, :] if indexes is not None else self.positive_triples
        return engine.ns_score(model.model_name, model._ent, model._rel, tri, neg, self.slot, False, model.l_norm)

    def score_with_positive(self, model: KgeModel) -> torch.Tensor:
        """[n, 1+K] assembly of train_negative_sampling.py:139-148 in one call."""
        return engine.ns_score(model.model_name, model._ent, model._rel, self.positive_triples, self._samples,
                               self.slot, True, model.l_norm)


# -- EntityRankingJob rank arithmetic (eval_entity_ranking.py:533-618) -------------------------------
def get_ranks_and_num_ties(scores, true_scores, rtol=1e-4, atol=1e-5):
    return engine.rank_dense(scores, true_scores, None, rtol, atol)


def filter_and_rank(scores_sp, scores_po, labels, o_true_scores, s_true_scores, rtol=1e-4, atol=1e-5):
    """Returns s_rank, s_num_ties, o_rank, o_num_ties (the filtered score copies are not produced)."""
    c = scores_sp.shape[1]
    lsp = labels[:, :c] if labels is not None else None
    lpo = labels[:, c:] if labels is not None else None
    o_rank, o_ties = engine.rank_dense(scores_sp, o_true_scores, lsp, rtol, atol)
    s_rank, s_ties = engine.rank_dense(scores_po, s_true_scores, lpo, rtol, atol)
    return s_rank, s_ties, o_rank, o_ties


def get_ranks(rank, num_ties, tie_handling="rounded_mean_rank"):
    if tie_handling == "rounded_mean_rank":
        return rank + num_ties // 2
    if tie_handling == "best_rank":
        return rank
    if tie_handling == "worst_rank":
        return rank + num_ties - 1
    raise NotImplementedError
