"""Golden vectors of the negative-sampling losses, from the LIVE reference's KgeLoss classes (kge/util/loss.py).

    python tests/golden/gen_ns_losses.py       # writes tests/golden/ns_losses.npz

Each case is one seeded [n, 1+K] score block (fp32 values) with one positive per row — in column 0 as the
negative-sampling job builds it (train_negative_sampling.py:126-137), or at a random column (the index-label form
the standalone KgeLoss mirror accepts).  The reference's loss runs on the block as
`KgeLoss.create(config)(scores, labels, num_negatives=K)` with a 0/1 label matrix, in fp64 (so rows with |z| >= 100 are
exact, where the reference's own fp32 soft-margin overflows); its value and autograd dL/dscores are stored.  Cases:
every loss; offset 0 and 2 for the BCE family; temperature 1 and 0.5 for bce_self_adversarial; margin 1 and 0 with an
exact tie (one negative equal to the positive); K in {1, 7, 1000}; moderate rows and rows with |z| >= 100.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

LOSSES = ("bce", "kl", "bce_mean", "bce_self_adversarial", "margin_ranking", "soft_margin", "se")


def _make(loss, arg, temperature):
    from kge import Config
    from kge.util.loss import KgeLoss

    c = Config()
    c.folder = None
    c.set("console.quiet", True)
    c.set("job.device", "cpu")
    c.set("train.type", "negative_sampling")
    c.set("train.loss", loss)
    c.set("train.loss_arg", arg)
    if loss == "bce_self_adversarial":
        c.set("user.bce_self_adversarial_temperature", temperature, create=True)
    return KgeLoss.create(c)


def cases():
    for loss in LOSSES:
        args = {"margin_ranking": (1.0, 0.0)}.get(loss, (0.0, 2.0) if loss.startswith("bce") else (float("nan"),))
        temps = (1.0, 0.5) if loss == "bce_self_adversarial" else (1.0,)
        for arg in args:
            for temp in temps:
                for K in (1, 7, 1000):
                    for big in (False, True):
                        yield loss, arg, temp, K, big


def main():
    ref_shim.import_reference()
    g = torch.Generator().manual_seed(2024)
    out = {}
    meta_loss, meta_arg, meta_temp = [], [], []
    for j, (loss, arg, temp, K, big) in enumerate(cases()):
        n = 2 if K == 1000 else 6
        m = 1 + K
        if big:   # |z| in [100, 150), random signs
            z = (100.0 + 50.0 * torch.rand((n, m), generator=g)) * torch.sign(torch.randn((n, m), generator=g))
        else:
            z = torch.randn((n, m), generator=g) * 3.0
        lab = torch.randint(0, m, (n,), generator=g) if K == 7 else torch.zeros(n, dtype=torch.long)
        if loss == "margin_ranking" and m > 2:      # an exact tie: one negative scored like the row's positive
            tie = (lab + 1) % m
            z[torch.arange(n), tie] = z[torch.arange(n), lab]
        z = z.float()
        y = torch.zeros((n, m), dtype=torch.float64)
        y[torch.arange(n), lab] = 1.0
        x = z.double().requires_grad_(True)
        value = _make(loss, arg, temp)(x, y, num_negatives=K)
        (grad,) = torch.autograd.grad(value, x)
        out[f"z_{j}"] = z.numpy()
        out[f"lab_{j}"] = lab.numpy()
        out[f"loss_{j}"] = np.float64(value.item())
        out[f"grad_{j}"] = grad.float().numpy()
        # the argument the loss ran with (the reference's NaN defaults resolved, loss.py:46-82)
        meta_loss.append(loss)
        meta_arg.append({"margin_ranking": arg}.get(loss, 0.0 if np.isnan(arg) else arg))
        meta_temp.append(temp)
    out["loss_name"] = np.array(meta_loss)
    out["arg"] = np.array(meta_arg, dtype=np.float64)
    out["temperature"] = np.array(meta_temp, dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "ns_losses.npz"), **out)
    print("wrote ns_losses.npz:", len(meta_loss), "cases")


if __name__ == "__main__":
    main()
