"""TEST INFRASTRUCTURE: embedding dropout of the negative-sampling step (kge_b200/csrc/ns_dropout.cu, layout in
include/b200kge.h) restated on the CPU mirror of tests/dropout_oracle.py: the masked [n, 1+K] block of one slot for the
`triple` and `batch` implementations in any dtype, and dropout modules that make the UNMODIFIED reference negative-
sampling job draw the mirror's masks under the plugin's keys."""
from __future__ import annotations

import contextlib

import torch

import dropout_oracle as dro

S, P, O = 0, 1, 2


def stream(slot, j):
    """Mask stream of draw j (0-2: the positive's s, p, o; 3-5: the negatives' s, p, o) of `slot`."""
    return 6 + 6 * slot + j


def mask_rows(p, key, strm, rows, dim):
    """Keep mask (bool) of the given global mask rows (any order, repeats allowed)."""
    rows = torch.as_tensor(rows).long().reshape(-1)
    if rows.numel() == 0:
        return torch.zeros((0, dim), dtype=torch.bool)
    lo, hi = int(rows.min()), int(rows.max()) + 1
    return dro.mask(p, key.seed, key.call, strm, hi - lo, dim, lo)[rows - lo]


def apply_rows(x, p, key, strm, rows):
    """x [len(rows), dim] with the masks of global mask rows `rows`, kept values scaled as the kernels do."""
    if p == 0:
        return x
    m = mask_rows(p, key, strm, rows, x.shape[1]).to(x.device)
    return torch.where(m, x * dro.scale(p), torch.zeros((), dtype=x.dtype, device=x.device))


def score_spo(model, s, p, o, l_norm=1.0, eps=True):
    """Row-wise score of gathered (masked) rows: score_spo of the reference for every in-scope model, with TransE's
    pairwise_distance eps (transe.py:18) when `eps`, and RotatE's modulus taken with gradient 0 at 0 (the kernels'
    convention; the reference's sqrt gives NaN there, and dropout makes such ties common)."""
    D = s.shape[1]
    h = D // 2
    if model == "distmult":
        return (s * p * o).sum(1)
    if model == "complex":
        sr, si, pr, pi, orr, oi = s[:, :h], s[:, h:], p[:, :h], p[:, h:], o[:, :h], o[:, h:]
        return (sr * pr * orr + si * pr * oi + sr * pi * oi - si * pi * orr).sum(1)
    if model == "simple":
        return 0.5 * (s[:, :h] * p[:, :h] * o[:, h:] + s[:, h:] * p[:, h:] * o[:, :h]).sum(1)
    if model == "cp":
        return (s[:, :h] * p * o[:, h:]).sum(1)
    if model == "rescal":
        M = p.view(-1, D, D)
        return torch.einsum("nr,nrc,nc->n", s, M, o)
    if model == "transe":
        d = s + p - o + (1e-6 if eps else 0.0)
        return -d.abs().sum(1) if l_norm == 1.0 else -d.pow(2).sum(1).sqrt()
    if model == "rotate":
        c, sn = torch.cos(p), torch.sin(p)
        qr, qi = s[:, :h] * c - s[:, h:] * sn, s[:, :h] * sn + s[:, h:] * c
        m2 = (qr - o[:, :h]) ** 2 + (qi - o[:, h:]) ** 2
        nz = m2 > 0
        return -(torch.where(nz, m2, torch.ones_like(m2)).sqrt() * nz).sum(1)
    raise ValueError(model)


def block(model, ent, rel, triples, slot, neg, key, implementation, l_norm=1.0):
    """The slot's [n, 1+K] block (positive first) under the six draws of `key`, in ent's dtype, differentiable in
    ent / rel."""
    tri = triples.long().cpu()
    neg = neg.long().cpu()
    n, K = neg.shape
    rb = key.row_base
    pe, pr = key.p_ent, key.p_rel
    i = torch.arange(n) + rb
    ops = []
    for c, (tab, pc) in enumerate(((ent, pe), (rel, pr), (ent, pe))):
        ops.append(apply_rows(tab[tri[:, c]], pc, key, stream(slot, c), i))
    pos = score_spo(model, *ops, l_norm=l_norm)
    if K == 0:
        return pos[:, None]
    t = tri.repeat_interleave(K, 0).clone()
    t[:, slot] = neg.reshape(-1)
    ops = []
    for c, (tab, pc) in enumerate(((ent, pe), (rel, pr), (ent, pe))):
        if implementation == "triple":
            rows = (rb + torch.arange(n)).repeat_interleave(K) * K + torch.arange(K).repeat(n)
        elif c == slot:
            rows = t[:, c]                                   # batch / all: the entity id
        else:
            rows = i.repeat_interleave(K)
        ops.append(apply_rows(tab[t[:, c]], pc, key, stream(slot, 3 + c), rows))
    negs = score_spo(model, *ops, l_norm=l_norm, eps=implementation == "triple").view(n, K)
    return torch.cat([pos[:, None], negs], 1)


# ---- the reference job with the mirror's masks -------------------------------------------------------------------
class _Holder:
    key = None
    K = 1
    slot = 0
    in_sampler = False
    phase = "pos"          # "pos" | "triple" | "batch"
    ids = None             # batch: the open slot's entity ids, in embed order
    spo_calls = 0

    def begin(self, slot, phase):
        self.slot, self.phase = slot, phase
        self.count = {"ent": 0, "rel": 0}


class MirrorDropout(torch.nn.Module):
    """Stands in for an embedder's torch.nn.Dropout and applies the mirror's mask of the call's draw.  Entity calls in
    the reference's order: score_spo embeds s then o (kge_model.py:663-680), score_sp embeds s then the targets, score_po
    embeds the targets, then o (kge_model.py:719-723); the relation is embedded once per call."""

    def __init__(self, p, holder, kind):
        super().__init__()
        self.p, self.holder, self.kind = p, holder, kind

    def forward(self, x):
        h = self.holder
        i = h.count[self.kind]
        h.count[self.kind] += 1
        k, rb, n, K = h.key, h.key.row_base, x.shape[0], h.K
        # score_spo: s then o; score_po: the targets (S) then o; score_sp: s then the targets (O)
        col = P if self.kind == "rel" else (S, O)[i]
        j = col if h.phase == "pos" else 3 + col
        if h.phase == "pos":
            rows = torch.arange(n) + rb
        elif h.phase == "triple":
            rows = torch.arange(n) + rb * K
        elif col == h.slot:
            rows = h.ids
        else:
            rows = torch.arange(n) + rb
        return apply_rows(x, self.p, k, stream(h.slot, j), rows)


def _in_sampler(score, holder):
    def wrapped(*a, **kw):
        holder.in_sampler = True
        try:
            return score(*a, **kw)
        finally:
            holder.in_sampler = False
    return wrapped


def patch_reference_ns_job(job, p_ent, p_rel):
    """Make an UNMODIFIED reference negative-sampling job draw the mirror's masks with the plugin's keys: the embedders'
    dropout modules are replaced, score_spo / score_sp / score_po mark the draw, and _process_subbatch sets the key."""
    from kge_b200 import engine
    from kge_b200.plugin.jobs import dropout_call

    holder = _Holder()
    model = job.model
    model.get_s_embedder().dropout = MirrorDropout(p_ent, holder, "ent")
    model.get_p_embedder().dropout = MirrorDropout(p_rel, holder, "rel")
    spo, sp, po = model.score_spo, model.score_sp, model.score_po

    def score_spo(s, p, o, direction=None):
        # the job scores the positive column itself; the `triple` negatives come from BatchNegativeSample.score
        holder.begin("spo".index(direction), "triple" if holder.in_sampler else "pos")
        return spo(s, p, o, direction=direction)

    def score_sp(s, p, o=None):
        holder.begin(O, "batch")
        holder.ids = torch.arange(job.dataset.num_entities()) if o is None else o.long().cpu()
        return sp(s, p, o)

    def score_po(p, o, s=None):
        holder.begin(S, "batch")
        holder.ids = torch.arange(job.dataset.num_entities()) if s is None else s.long().cpu()
        return po(p, o, s)

    model.score_spo, model.score_sp, model.score_po = score_spo, score_sp, score_po
    orig = job._process_subbatch
    state = {}

    def process(batch_index, batch, subbatch_slice, result):
        pos = (job.epoch, batch_index)
        ordinal = state["ordinal"] + 1 if state.get("pos") == pos else 0
        state.update(pos=pos, ordinal=ordinal)
        holder.key = engine.DropoutKey(p_ent, p_rel, torch.initial_seed(), dropout_call(job.epoch, batch_index, ordinal),
                                       subbatch_slice.start or 0)
        holder.K = max(job._sampler.num_samples)
        for sample in batch["negative_samples"]:
            if sample is not None and not getattr(sample, "_mirror_marked", False):
                sample.score = _in_sampler(sample.score, holder)
                sample._mirror_marked = True
        return orig(batch_index, batch, subbatch_slice, result)

    job._process_subbatch = process
    return job


# ---- engine stand-ins (CPU) that accept a dropout key -----------------------------------------------------------------
calls = {"dropout": 0}


def _ns_score(model, ent, rel, triples, negatives, slot, with_positive=False, l_norm=1.0, dropout=None,
              implementation="batch"):
    import engine_stub

    if dropout is None:
        return engine_stub.ns_score(model, ent, rel, triples, negatives, slot, with_positive, l_norm)
    calls["dropout"] += 1
    return block(model, ent, rel, triples, slot, negatives, dropout, implementation, l_norm).detach()


def _ns_loss(scores, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None, want_grad=False,
             return_rows=False):
    import ns_loss_oracle as nlo

    value = nlo.ns_loss(scores, loss, arg, temperature, label_idx, batch_size)
    G = nlo.ns_loss_grad(scores, loss, arg, temperature, label_idx, batch_size) if want_grad else None
    if return_rows:
        return value, G, nlo.ns_loss_rows(scores, loss, arg, temperature, label_idx)
    return value, G


def _ns_backward(model, ent, rel, triples, negatives, offset=0.0, l_norm=1.0, batch_size=None, grad_scores=None,
                 dropout=None, implementation="batch"):
    import engine_stub

    if dropout is None:
        return engine_stub.ns_backward(model, ent, rel, triples, negatives, offset, l_norm, batch_size)
    calls["dropout"] += 1
    e, r = ent.detach().clone().requires_grad_(True), rel.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        total = sum((grad_scores[sl] * block(model, e, r, triples, sl, neg, dropout, implementation, l_norm)).sum()
                    for sl, neg in negatives.items())
        de, dr = torch.autograd.grad(total, (e, r))
    return de, dr


@contextlib.contextmanager
def installed():
    """dropout_oracle.installed() plus CPU stand-ins of ns_score / ns_loss / ns_backward that apply the mirror's masks
    when given a dropout key; calls["dropout"] counts the calls that received one."""
    from kge_b200 import engine

    repl = {"ns_score": _ns_score, "ns_loss": _ns_loss, "ns_backward": _ns_backward}
    with dro.installed():
        saved = {k: getattr(engine, k) for k in repl}
        for k, v in repl.items():
            setattr(engine, k, v)
        try:
            yield
        finally:
            for k, v in saved.items():
                setattr(engine, k, v)
