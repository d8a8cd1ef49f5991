"""One shared-negative-sampling training batch, `user.b200_ns_shared` on vs off (H100).

Workload: the recipe LibKGE's README gives for its large graphs: B200TrainingJobNegativeSampling, batch 1024, D = 128,
num_samples s = o = 1000 shared (`shared_type: default`, `with_replacement: True`), kl, `implementation: batch`,
Adagrad with `lookup_embedder.sparse: True`; one batch = forward + backward (job._process_batch) + the optimizer step.
Shapes Yago3-10 (E = 123,182, R = 37) and Wikidata5M-sized (E = 4.8 M, R = 822); models ComplEx and RotatE L1.  Arms:
the option on (each slot scored against its U' shared rows, b200kge_ns_shared_*) and off (today's route: the per-row
[n, K] ids through ns_kernel / ns_backward_kernel), fed the same host-drawn batch, alternated, median of --reps.  Both
arms start from identical tables; their losses on the batch are compared.  With --profile one batch of each arm runs
under torch.profiler and the CUDA time of its kernels is listed.  The card's name and power limit are read in the same
run.
Usage: python scripts/ns_shared_train_bench.py [--reps 7] [--profile] [--out file.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from kge_b200 import hostenv  # noqa: E402

N, D, K = 1024, 128, 1000
SHAPES = {"yago3-10": (123182, 37), "wikidata5m": (4_800_000, 822)}
CASES = [("complex", 1.0), ("rotate", 1.0)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0].split(", ")
    return q[0], q[1]


def make_job(model, ln, E, R, option, triples):
    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import Job

    name = "b200_" + model
    c = Config()
    c.folder = tempfile.mkdtemp()
    c.set("console.quiet", True)
    c.set("modules", ["kge.job", "kge.model", "kge.model.embedder", "kge_b200.plugin"])
    c.set("model", name)
    c._import(name)
    for k, v in {"dataset.name": "bench", "dataset.num_entities": E, "dataset.num_relations": R,
                 "dataset.pickle": False, "job.device": "cuda", "job.type": "train",
                 "train.type": "negative_sampling", "train.loss": "kl", "train.batch_size": N,
                 "train.optimizer.default.type": "Adagrad",
                 "negative_sampling.class_name": "B200TrainingJobNegativeSampling",
                 "negative_sampling.implementation": "batch", "negative_sampling.num_samples.s": K,
                 "negative_sampling.num_samples.o": K, "negative_sampling.shared": True,
                 "negative_sampling.shared_type": "default", "negative_sampling.with_replacement": True,
                 "user.b200_ns_shared": option}.items():
        c.set(k, v)
    c.set_all({"lookup_embedder.dim": D, "lookup_embedder.sparse": True})
    if model in ("transe", "rotate"):
        c.set(name + ".l_norm", ln)
    ds = Dataset(c, None)
    ds._triples = {"train": triples, "valid": triples[:10], "test": triples[:10]}
    ds._meta = {"entity_ids": [f"e{i}" for i in range(E)], "relation_ids": [f"r{i}" for i in range(R)]}
    job = Job.create(c, ds)
    job._prepare()
    return job


def run_batch(job, batch):
    job.optimizer.zero_grad(set_to_none=True)
    res = job._process_batch(0, batch)
    job.optimizer.step()
    return res.avg_loss


def kernel_times(job, batch, top=14):
    """CUDA time (ms) of one batch per kernel (the `top` longest) and in all."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_batch(job, batch)
        torch.cuda.synchronize()
    rows = sorted(((ev.key[:70], ev.device_time_total / 1e3) for ev in prof.key_averages()
                   if ev.device_time_total > 0), key=lambda r: -r[1])
    return {"total": round(sum(t for _, t in rows), 4), "kernels": {k: round(t, 4) for k, t in rows[:top]}}


def one_case(model, ln, E, R, reps, profile):
    g = torch.Generator().manual_seed(0)
    tri = torch.stack([torch.randint(0, E, (4 * N,), generator=g), torch.randint(0, R, (4 * N,), generator=g),
                       torch.randint(0, E, (4 * N,), generator=g)], 1).int()
    row = {"model": model if model == "complex" else f"{model} L{int(ln)}", "E": E, "R": R}
    jobs = {}
    try:
        for arm in ("on", "off"):
            jobs[arm] = make_job(model, ln, E, R, arm == "on", tri)
        with torch.no_grad():
            for a, b in zip(jobs["on"].model.parameters(), jobs["off"].model.parameters()):
                b.copy_(a)
        torch.manual_seed(7)
        batch = jobs["on"]._get_collate_fun()(list(range(N)))       # one shared draw serves both arms
        row["num_unique_s_o"] = [len(batch["negative_samples"][slot]._unique_samples) for slot in (0, 2)]
        losses = {arm: run_batch(job, batch) for arm, job in jobs.items()}      # also the warm-up
        row["loss_on"], row["loss_off"] = losses["on"], losses["off"]
        row["loss_rel_diff"] = abs(losses["on"] - losses["off"]) / max(abs(losses["off"]), 1e-30)
        times = {arm: [] for arm in jobs}
        for _ in range(reps):
            for arm, job in jobs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run_batch(job, batch)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) * 1e3)
        row["on_ms"], row["off_ms"] = statistics.median(times["on"]), statistics.median(times["off"])
        row["on_range_ms"] = [min(times["on"]), max(times["on"])]
        row["off_range_ms"] = [min(times["off"]), max(times["off"])]
        row["speedup"] = row["off_ms"] / row["on_ms"]
        if profile:
            row["profile_ms"] = {arm: kernel_times(job, batch) for arm, job in jobs.items()}
    except RuntimeError as e:            # torch.cuda.OutOfMemoryError
        if "out of memory" not in str(e):
            raise
        row["oom"] = next(line for line in str(e).splitlines() if "out of memory" in line).strip()
    finally:
        jobs.clear()
        torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    rows = []
    for shape, (E, R) in SHAPES.items():
        for model, ln in CASES:
            row = dict(shape=shape, **one_case(model, ln, E, R, a.reps, a.profile))
            print(json.dumps(row), flush=True)
            rows.append(row)
    res = {"card": name, "power_limit": power, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
