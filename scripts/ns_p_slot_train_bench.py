"""One negative-sampling training batch with a sampled P slot, `user.b200_ns_p_slot` on vs off (H100).

Workload: B200TrainingJobNegativeSampling, 512 triples, num_samples s = o = 1000 and p = 100 (one ComplEx row at
p = 1000), kl, d = 512, `implementation: batch`, uniform negatives drawn on the host; one batch = forward + backward
(job._process_batch), no optimizer step.  Shapes FB15k-237 (E = 14,541, R = 237) and WN18RR (E = 40,943, R = 11); models
ComplEx, TransE L1, RotatE L1.  Arms: the option on (S, P and O slots native) and off (today's route: the reference
step of the whole sub-batch on the same plugin model), alternated, median of --reps.  Both arms start from identical
tables and their losses on the same batch are compared.  An arm that runs out of memory is reported as such.  With
--profile a torch.profiler run of the option-on arm splits the P slot's time between its forward (spo_kernel) and the
kernels of its backward.  The card's name and power limit are read in the same run.
Usage: python scripts/ns_p_slot_train_bench.py [--reps 7] [--profile] [--out file.json]
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

N, D, KSO = 512, 512, 1000
SHAPES = {"fb15k-237": (14541, 237), "wn18rr": (40943, 11)}
CASES = [("complex", 1.0, 100), ("transe", 1.0, 100), ("rotate", 1.0, 100), ("complex", 1.0, 1000)]
# kernels of the P slot's backward (b200kge_ns_p_backward): its own, the s_o fold / unfold and the GEMM block
P_BACKWARD = ("ns_p_", "fold_so", "unfold_so", "transpose", "presplit", "gemm", "pairwise_tc")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0].split(", ")
    return q[0], q[1]


def make_job(model, ln, E, R, kp, option, triples):
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
                 "negative_sampling.class_name": "B200TrainingJobNegativeSampling",
                 "negative_sampling.implementation": "batch", "negative_sampling.num_samples.s": KSO,
                 "negative_sampling.num_samples.o": KSO, "negative_sampling.num_samples.p": kp,
                 "user.b200_ns_p_slot": option}.items():
        c.set(k, v)
    c.set_all({"lookup_embedder.dim": D})
    if model in ("transe", "rotate"):
        c.set(name + ".l_norm", ln)
    ds = Dataset(c, None)
    ds._triples = {"train": triples, "valid": triples[:10], "test": triples[:10]}
    ds._meta = {"entity_ids": [f"e{i}" for i in range(E)], "relation_ids": [f"r{i}" for i in range(R)]}
    job = Job.create(c, ds)
    job._prepare()
    return job


def run_batch(job, batch):
    job.model.zero_grad(set_to_none=True)
    res = job._process_batch(0, batch)
    return res.avg_loss


def one_case(model, ln, kp, E, R, reps, profile):
    g = torch.Generator().manual_seed(0)
    tri = torch.stack([torch.randint(0, E, (4 * N,), generator=g), torch.randint(0, R, (4 * N,), generator=g),
                       torch.randint(0, E, (4 * N,), generator=g)], 1).int()
    row = {"model": f"{model} L{int(ln)}" if model != "complex" else model, "E": E, "R": R, "num_samples_p": kp}
    jobs = {}
    try:
        for arm in ("on", "off"):
            jobs[arm] = make_job(model, ln, E, R, kp, arm == "on", tri)
        with torch.no_grad():
            for a, b in zip(jobs["on"].model.parameters(), jobs["off"].model.parameters()):
                b.copy_(a)
        torch.manual_seed(7)
        batch = jobs["on"]._get_collate_fun()(list(range(N)))
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
        row["speedup"] = row["off_ms"] / row["on_ms"]
        if profile:
            row["p_slot_profile_ms"] = p_slot_profile(jobs["on"], batch)
    except RuntimeError as e:            # torch.cuda.OutOfMemoryError, or one raised inside a TorchScript function
        if "out of memory" not in str(e):
            raise
        row["oom"] = next(line for line in str(e).splitlines() if "out of memory" in line).strip()
    finally:
        jobs.clear()
        torch.cuda.empty_cache()
    return row


def p_slot_profile(job, batch):
    """CUDA time (ms) of one option-on batch by kernel group: the P slot's forward (spo_kernel) and its backward."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_batch(job, batch)
        torch.cuda.synchronize()
    out = {"p_forward_spo_kernel": 0.0, "p_backward": 0.0, "other": 0.0}
    kernels = {}
    for ev in prof.key_averages():
        t = ev.device_time_total / 1e3
        if t <= 0:
            continue
        if "spo_kernel" in ev.key:
            out["p_forward_spo_kernel"] += t
        elif any(k in ev.key for k in P_BACKWARD):
            out["p_backward"] += t
            kernels[ev.key[:60]] = round(t, 4)
        else:
            out["other"] += t
    out["p_backward_kernels"] = kernels
    return out


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
        for model, ln, kp in CASES:
            row = dict(shape=shape, **one_case(model, ln, kp, E, R, a.reps, a.profile))
            print(json.dumps(row), flush=True)
            rows.append(row)
    res = {"card": name, "power_limit": power, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
