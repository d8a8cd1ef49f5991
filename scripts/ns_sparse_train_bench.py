"""One negative-sampling training batch with the optimizer step, dense vs row-sparse table gradients (H100).

Workload: ComplEx d=512, S and O slots, K = 1000 uniform negatives drawn on the device, 512 triples, kl; forward,
backward through the plugin's _NsSlotLossFn, optimizer.step() and zero_grad(), at E = 40,943 and E = 4.8M (R = 237).
Arms, median of --reps: `sparse: False` with Adagrad (dense gradients, dense step) alternated with `sparse: True` with
Adagrad (b200kge_ns_backward_sparse, row-sparse step); then `sparse: True` with SparseAdam.  The two Adagrad arms start from
the same tables and take the same seeded batch once more after the timing; the max difference of the updated tables is
printed.  The card's name and power limit are read in the same run.  Usage: python scripts/ns_sparse_train_bench.py
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from kge_b200 import engine, hostenv  # noqa: E402

D, R, N, K = 512, 237, 512, 1000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0].split(", ")
    return q[0], q[1]


class _Model:
    """What _NsSlotLossFn reads of a plugin model."""
    _b200_name = "complex"

    def __init__(self, sparse):
        self.sparse = sparse

    def _b200_args(self):
        return 1.0, "auto"

    def b200_sparse_grads(self):
        return (self.sparse, self.sparse)


def make_arm(E, sparse, opt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ent = torch.nn.Parameter(torch.randn(E, D, device="cuda", generator=g) * 0.1)
    rel = torch.nn.Parameter(torch.randn(R, D, device="cuda", generator=g) * 0.1)
    o = torch.optim.Adagrad([ent, rel], lr=0.1) if opt == "adagrad" else torch.optim.SparseAdam([ent, rel], lr=1e-3)
    return ent, rel, o, _Model(sparse)


def batch(E, i):
    gen = torch.Generator(device="cuda").manual_seed(1000 + i)
    tri = torch.stack([torch.randint(0, E, (N,), device="cuda", generator=gen),
                       torch.randint(0, R, (N,), device="cuda", generator=gen),
                       torch.randint(0, E, (N,), device="cuda", generator=gen)], 1)
    return tri


def step(arm, E, i):
    hostenv.import_kge()
    from kge_b200.plugin import _NsSlotLossFn

    ent, rel, opt, model = arm
    tri = batch(E, i)
    for slot in (0, 2):
        neg = engine.sample_uniform(N, K, E, 5, (i << 2) | slot, "cuda")
        loss = _NsSlotLossFn.apply(ent, rel, model, tri, neg, slot, 0.0, N, "kl", 1.0, None, "batch")
        loss.item()                       # the job reads every slot's loss
        loss.backward()
    opt.step()
    opt.zero_grad()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="40943,4800000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for E in (int(x) for x in a.sizes.split(",")):
        # the two Adagrad arms alternated; the SparseAdam arm afterwards on its own (at E = 4.8M the three arms' tables,
        # optimizer states and dense gradients do not fit in 80 GB together)
        times = {}
        for group in (("dense_adagrad", "sparse_adagrad"), ("sparse_sparseadam",)):
            arms = {k: make_arm(E, k.startswith("sparse"), k.split("_")[1]) for k in group}
            for arm in arms.values():        # warm-up: modules, allocator, optimizer state
                step(arm, E, 0)
            torch.cuda.synchronize()
            for k in arms:
                times[k] = []
            for r in range(a.reps):
                for k, arm in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    step(arm, E, 1 + r)
                    torch.cuda.synchronize()
                    times[k].append((time.perf_counter() - t0) * 1e3)
            del arms
            torch.cuda.empty_cache()
        # the Adagrad arms from identical tables and state through one more identical batch
        fresh = {k: make_arm(E, k.startswith("sparse"), "adagrad", seed=3) for k in ("dense_adagrad", "sparse_adagrad")}
        for arm in fresh.values():
            step(arm, E, 99)
        torch.cuda.synchronize()
        de = float((fresh["dense_adagrad"][0] - fresh["sparse_adagrad"][0]).abs().max())
        dr = float((fresh["dense_adagrad"][1] - fresh["sparse_adagrad"][1]).abs().max())
        row = {"E": E, **{k + "_ms": statistics.median(v) for k, v in times.items()},
               "adagrad_max_abs_diff_ent": de, "adagrad_max_abs_diff_rel": dr}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del fresh
        torch.cuda.empty_cache()
    res = {"card": name, "power_limit": power, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
