"""torch's optimizer step against the native one (kge_b200.optim) in a training batch (H100).

Workload: the batch of scripts/ns_sparse_train_bench.py (ComplEx d=512, S and O slots, K = 1000 negatives drawn on the
device, 512 triples, kl; forward and backward through the plugin's _NsSlotLossFn, optimizer.step(), zero_grad()) at
E = 40,943 and E = 4.8M (R = 237), for three arm pairs: dense Adagrad, sparse Adagrad (`sparse: True`) and SparseAdam.
Each pair is torch's step and the native step from identical tables, alternated, median of --reps; the whole batch is
timed with a host clock around synchronised work and the step alone with CUDA events.  After the timed batches (the same
seeded batches for both arms) the max table difference between the arms is printed.  Also: the 1vsAll headline batch
(E = 14,541, n = 1024, bce, engine.train_1vsall_forward / _backward) with a dense Adagrad step, and the dense kernel
alone at E rows, as achieved bytes/s (20 B per element) over 3.35 TB/s.

`--profile` (a separate run) records one sparse-Adagrad batch per size with torch's step under torch.profiler and prints
the CUDA time per kernel.  The card's name and power limit are read in the same run.
Usage: python scripts/native_optim_bench.py [--profile] [--out FILE]
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

from kge_b200 import engine, hostenv, optim  # noqa: E402

D, R, N, K = 512, 237, 512, 1000
HBM = 3.35e12


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


def make_arm(E, kind, native, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ent = torch.nn.Parameter(torch.randn(E, D, device="cuda", generator=g) * 0.1)
    rel = torch.nn.Parameter(torch.randn(R, D, device="cuda", generator=g) * 0.1)
    o = torch.optim.SparseAdam([ent, rel], lr=1e-3) if kind == "sparse_adam" else torch.optim.Adagrad([ent, rel], lr=0.1)
    if native:
        optim.install_native_step(o)
    return ent, rel, o, _Model(kind != "dense_adagrad")


def ns_forward_backward(arm, E, i):
    hostenv.import_kge()
    from kge_b200.plugin import _NsSlotLossFn

    ent, rel, opt, model = arm
    gen = torch.Generator(device="cuda").manual_seed(1000 + i)
    tri = torch.stack([torch.randint(0, E, (N,), device="cuda", generator=gen),
                       torch.randint(0, R, (N,), device="cuda", generator=gen),
                       torch.randint(0, E, (N,), device="cuda", generator=gen)], 1)
    for slot in (0, 2):
        neg = engine.sample_uniform(N, K, E, 5, (i << 2) | slot, "cuda")
        loss = _NsSlotLossFn.apply(ent, rel, model, tri, neg, slot, 0.0, N, "kl", 1.0, None, "batch")
        loss.item()                       # the job reads every slot's loss
        loss.backward()


def ns_batch(arm, E, i, ev=None):
    ns_forward_backward(arm, E, i)
    opt = arm[2]
    if ev:
        ev[0].record()
    opt.step()
    if ev:
        ev[1].record()
    opt.zero_grad()


def same_grad_diff(make, forward_backward):
    """Max table difference after one step of torch's and of the native step from identical tables, state and
    gradients (the gradients of one batch, computed once)."""
    a = make(False)
    forward_backward(a)
    grads = [p.grad.clone() for p in a[:2]]
    a[2].step()
    want = [p.detach() for p in a[:2]]
    del a
    b = make(True)
    for p, g in zip(b[:2], grads):
        p.grad = g
    del grads
    b[2].step()
    diff = max(float((x - y.detach()).abs().max()) for x, y in zip(want, b[:2]))
    del b, want
    torch.cuda.empty_cache()
    return diff


def time_pair(make, run, reps):
    """{arm: (batch ms, step ms)} medians, torch's and the native step alternated, and the max table difference of the
    two arms after the timed batches (the backward's atomics make their gradients differ in the last bits)."""
    arms = {"torch": make(False), "native": make(True)}
    for arm in arms.values():             # warm-up: modules, allocator, optimizer state
        run(arm, 0, None)
    torch.cuda.synchronize()
    times = {k: ([], []) for k in arms}
    for r in range(reps):
        for k, arm in arms.items():
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(arm, 1 + r, ev)
            torch.cuda.synchronize()
            times[k][0].append((time.perf_counter() - t0) * 1e3)
            times[k][1].append(ev[0].elapsed_time(ev[1]))
    diff = max(float((a - b).abs().max()) for a, b in zip(arms["torch"][:2], arms["native"][:2]))
    out = {k: (statistics.median(v[0]), statistics.median(v[1])) for k, v in times.items()}
    del arms
    torch.cuda.empty_cache()
    return out, diff


def onevsall_pair(reps):
    E1, n = 14541, 1024

    def make(native):
        g = torch.Generator(device="cuda").manual_seed(0)
        ent = torch.nn.Parameter(torch.randn(E1, D, device="cuda", generator=g) * 0.1)
        rel = torch.nn.Parameter(torch.randn(R, D, device="cuda", generator=g) * 0.1)
        o = torch.optim.Adagrad([ent, rel], lr=0.1)
        if native:
            optim.install_native_step(o)
        return ent, rel, o

    def forward_backward(arm, i):
        ent, rel, opt = arm
        gen = torch.Generator(device="cuda").manual_seed(2000 + i)
        tri = torch.stack([torch.randint(0, E1, (n,), device="cuda", generator=gen),
                           torch.randint(0, R, (n,), device="cuda", generator=gen),
                           torch.randint(0, E1, (n,), device="cuda", generator=gen)], 1)
        engine.train_1vsall_forward("complex", ent.detach(), rel.detach(), tri, "bce").item()
        d_ent, d_rel = engine.train_1vsall_backward("complex", ent.detach(), rel.detach(), tri, "bce")
        ent.grad, rel.grad = d_ent, d_rel

    def run(arm, i, ev):
        forward_backward(arm, i)
        opt = arm[2]
        if ev:
            ev[0].record()
        opt.step()
        if ev:
            ev[1].record()
        opt.zero_grad()
    t, diff = time_pair(make, run, reps)
    return t, diff, same_grad_diff(make, lambda arm: forward_backward(arm, 99))


def dense_kernel(E, iters=20):
    """The dense Adagrad kernel alone on [E, D]: ms per launch and achieved bytes/s (read p, g, sum; write p, sum)."""
    p, s, g = (torch.rand(E, D, device="cuda") for _ in range(3))
    for _ in range(3):
        engine.adagrad_step(p, s, g, 1e-3, 1e-10)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        engine.adagrad_step(p, s, g, 1e-3, 1e-10)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    rate = 20.0 * E * D / (ms * 1e-3)
    del p, s, g
    torch.cuda.empty_cache()
    return {"E": E, "kernel_ms": ms, "bytes_per_s": rate, "fraction_of_3.35TBps": rate / HBM}


def profile(sizes):
    from torch.profiler import ProfilerActivity, profile as prof

    out = []
    for E in sizes:
        arm = make_arm(E, "sparse_adagrad", False)
        ns_batch(arm, E, 0)
        torch.cuda.synchronize()
        row = {"E": E}
        # forward + backward (row sets, scoring, loss, scatter) and torch's step recorded apart
        for phase, fn in (("forward_backward", lambda: ns_forward_backward(arm, E, 1)), ("torch_step", arm[2].step)):
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                fn()
                torch.cuda.synchronize()
            kernels = {}
            for e in p.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    kernels[e.name] = kernels.get(e.name, 0.0) + e.device_time_total / 1e3
            top = sorted(kernels.items(), key=lambda kv: -kv[1])
            total = sum(kernels.values())
            print(f"E = {E}, {phase}: {total:.3f} ms of CUDA time in one sparse-Adagrad batch")
            for name, ms in top[:20]:
                print(f"  {ms:8.3f} ms  {name[:140]}")
            row[phase] = {"total_ms": total, "kernels": top}
        arm[2].zero_grad()
        out.append(row)
        del arm
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="40943,4800000")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    sizes = [int(x) for x in a.sizes.split(",")]
    if a.profile:
        res = {"card": name, "power_limit": power, "profile": profile(sizes)}
    else:
        rows = []
        for E in sizes:
            for kind in ("dense_adagrad", "sparse_adagrad", "sparse_adam"):
                make = lambda native: make_arm(E, kind, native)  # noqa: E731
                t, diff = time_pair(make, lambda arm, i, ev: ns_batch(arm, E, i, ev), a.reps)
                same = same_grad_diff(make, lambda arm: ns_forward_backward(arm, E, 99))
                row = {"E": E, "arms": kind, "batch_ms_torch": t["torch"][0], "batch_ms_native": t["native"][0],
                       "step_ms_torch": t["torch"][1], "step_ms_native": t["native"][1],
                       "max_table_diff_after_timed_batches": diff, "max_table_diff_same_grads": same}
                print(json.dumps(row), flush=True)
                rows.append(row)
        t, diff, same = onevsall_pair(a.reps)
        row = {"E": 14541, "arms": "1vsAll bce n=1024, dense_adagrad", "batch_ms_torch": t["torch"][0],
               "batch_ms_native": t["native"][0], "step_ms_torch": t["torch"][1], "step_ms_native": t["native"][1],
               "max_table_diff_after_timed_batches": diff, "max_table_diff_same_grads": same}
        print(json.dumps(row), flush=True)
        rows.append(row)
        kern = [dense_kernel(E) for E in sizes]
        for k in kern:
            print(json.dumps(k), flush=True)
        res = {"card": name, "power_limit": power, "rows": rows, "dense_kernel": kern}
    print(json.dumps({"card": name, "power_limit": power}))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
