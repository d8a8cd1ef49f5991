"""TEST INFRASTRUCTURE: CPU restatement of the negative-sampling losses and of their gradient (kge/util/loss.py), in the
dtype of the scores (fp32 or fp64), and the negative-sampling backward of oracle/kge_fold.py generalised to any of
them.

Every loss is a function of one [n, m] block with one positive per row (column label_idx[i], default 0; label 0
elsewhere, K = m - 1 negatives), summed over rows (the job divides by the batch size,
train_negative_sampling.py:156):

    bce                   sum_c bce(z_c + o, y_c)                                 loss.py:153-159
    kl                    lse(z) - z_l                                            loss.py:198-213
    bce_mean              (bce(z_l + o, 1) + sum_c bce(z_c + o, 0) / K) / 2       loss.py:160-168
    bce_self_adversarial  (bce(z_l + o, 1) + sum_c w_c bce(z_c + o, 0)) / 2,
                          w = softmax(T (z_c + o)) over the negatives, detached   loss.py:169-187
    margin_ranking        sum_c max(0, margin - z_l + z_c)                        loss.py:240-252
    soft_margin           sum_c log(1 + exp(-y_c z_c)), y = +1 | -1               loss.py:216-224
    se                    sum_c (z_c - y_c)^2                                     loss.py:267-274
"""
from __future__ import annotations

import torch

from oracle import kge_fold as kf

LOSSES = ("bce", "kl", "bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se")


def _softplus(x):
    return x.clamp_min(0) + torch.log1p(torch.exp(-x.abs()))


def _parts(z, label_idx):
    n, m = z.shape
    lab = torch.zeros(n, dtype=torch.long) if label_idx is None else label_idx.long().view(-1)
    y = torch.zeros_like(z)
    y[torch.arange(n), lab] = 1.0
    neg = y == 0
    zl = z[torch.arange(n), lab]
    return lab, y, neg, zl


def ns_loss_rows(z, loss, arg=0.0, temperature=1.0, label_idx=None):
    """Per-row losses [n] of the block z [n, m]."""
    lab, y, neg, zl = _parts(z, label_idx)
    o = arg
    m = z.shape[1]
    if loss == "bce":
        return _softplus(z + o).sum(1) - ((z + o) * y).sum(1)
    if loss == "kl":
        mx = z.max(1).values
        return (mx - zl) + torch.log(torch.exp(z - mx[:, None]).sum(1))
    pos_bce = _softplus(-(zl + o))
    if loss == "bce_mean":
        return 0.5 * (pos_bce + (_softplus(z + o) * neg).sum(1) / (m - 1))
    if loss == "bce_self_adversarial":
        w = _adversarial_weights(z, neg, o, temperature)
        return 0.5 * (pos_bce + (w * _softplus(z + o)).sum(1))
    if loss == "margin_ranking":
        return ((-(zl[:, None] - z) + o).clamp_min(0) * neg).sum(1)
    if loss == "soft_margin":
        return _softplus(-(2 * y - 1) * z).sum(1)
    if loss == "se":
        return ((z - y) ** 2).sum(1)
    raise ValueError(loss)


def _adversarial_weights(z, neg, o, temperature):
    t = torch.where(neg, temperature * (z + o), torch.full_like(z, -float("inf")))
    return torch.softmax(t, 1)


def ns_loss(z, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None):
    """Scalar loss: sum of the row losses / batch_size (1 if None)."""
    return ns_loss_rows(z, loss, arg, temperature, label_idx).sum() / (batch_size or 1)


def ns_loss_grad(z, loss, arg=0.0, temperature=1.0, label_idx=None, batch_size=None):
    """dL/dz [n, m] of ns_loss, analytic (what the row-loss kernel writes as G).  The margin-ranking hinge passes the
    gradient at exactly 0, as torch's clamp_min does; the self-adversarial weights are constants."""
    lab, y, neg, zl = _parts(z, label_idx)
    o = arg
    m = z.shape[1]
    sig = torch.sigmoid(z + o)
    if loss == "bce":
        g = sig - y
    elif loss == "kl":
        g = torch.softmax(z, 1) - y
    elif loss == "bce_mean":
        g = torch.where(neg, 0.5 * sig / (m - 1), 0.5 * (sig - 1))
    elif loss == "bce_self_adversarial":
        w = _adversarial_weights(z, neg, o, temperature)
        g = torch.where(neg, 0.5 * w * sig, 0.5 * (sig - 1))
    elif loss == "margin_ranking":
        act = ((-(zl[:, None] - z) + o) >= 0) & neg
        g = act.to(z.dtype)
        g[torch.arange(z.shape[0]), lab] = -act.sum(1).to(z.dtype)
    elif loss == "soft_margin":
        s = 2 * y - 1
        g = -s * torch.sigmoid(-s * z)
    elif loss == "se":
        g = 2 * (z - y)
    else:
        raise ValueError(loss)
    return g / (batch_size or 1)


def ns_backward(model, ent, rel, triples, negatives, loss="bce", arg=0.0, temperature=1.0, l_norm=1.0,
                batch_size=None):
    """(dEnt, dRel) of one negative-sampling batch with any loss above: per slot the [n, 1+K] block (positive first),
    loss summed and divided by batch_size (default n).  negatives = {slot: [n, K] ids}.  With loss="bce" this is
    oracle/kge_fold.ns_backward."""
    n = triples.shape[0]
    d_ent, d_rel = torch.zeros_like(ent), torch.zeros_like(rel)
    for slot, neg in negatives.items():
        k = neg.shape[1]
        t = triples.long().repeat_interleave(1 + k, 0).view(n, 1 + k, 3).clone()
        t[:, 1:, slot] = neg.long()
        t = t.view(-1, 3)
        z = kf.pair_rowwise(model, ent, rel, t[:, 0], t[:, 1], t[:, 2], l_norm).view(n, 1 + k)
        g = ns_loss_grad(z, loss, arg, temperature, None, batch_size or n).reshape(-1)
        kf.spo_backward(model, ent, rel, t[:, 0], t[:, 1], t[:, 2], g, d_ent, d_rel, l_norm)
    return d_ent, d_rel
