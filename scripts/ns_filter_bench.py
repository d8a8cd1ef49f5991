"""Time one negative-sampling training batch with filtered negatives (negative_sampling.filtering.s and .o), forward +
backward of the S and O slots, no optimizer step, two routes of B200TrainingJobNegativeSampling alternated in one
process:

  (a) host    the job as it runs without user.b200_device_sampling: the collate draws the negatives with torch.randint,
              filters them with the reference's `fast` filter (numba) and the step copies the ids to the device
  (b) device  user.b200_device_sampling: true — the collate slices the triples, b200kge_sample_uniform_filtered draws
              and filters on the device

Each timed batch is the collate of the batch's triples (with train.num_workers 0 it runs in the job's thread) plus
_process_batch, up to a device synchronise.  ComplEx, kl, d = 512, K = 1000 per slot, batch 512; triples from a seeded
split whose subjects and objects follow Zipf(1.0) (SURVEY 8(d)) so that heavy keys exist, at a WN18RR shape
(40,943 / 11 / 86,835) and an FB15k-237 shape (14,541 / 237 / 272,115).  Median of --reps after --warmup.  Also
reported: the sampling kernel's own time (CUDA events over 100 launches, both slots), the fraction of draws the filter
replaces, and the card's name and power limit.  The fraction is an estimate over the timed batch's triples: the numpy
mirror (tests/ns_filter_oracle.py) counts it for one draw of its own (seed 5, offset = slot), not for the timed draws.

    python scripts/ns_filter_bench.py [--reps 7] [--json OUT]

Needs the reference installed (oracle/install_ref.sh) and an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ns_train_bench import card  # noqa: E402

SHAPES = (("WN18RR", 40943, 11, 86835), ("FB15k-237", 14541, 237, 272115))
D, K, BATCH = 512, 1000, 512


def zipf_split(E, R, N, seed=0):
    """s, o ~ Zipf(1.0) over the entity ids (P(id) proportional to 1 / (id + 1)), p uniform."""
    g = torch.Generator().manual_seed(seed)
    w = 1.0 / torch.arange(1, E + 1, dtype=torch.float64)
    s = torch.multinomial(w, N, replacement=True, generator=g)
    o = torch.multinomial(w, N, replacement=True, generator=g)
    p = torch.randint(0, R, (N,), generator=g)
    return torch.stack([s, p, o], 1).int()


def make_job(E, R, split, device_sampling):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="ns_filter_bench_")
    config.set("console.quiet", True)
    config.set("modules", ["kge.job", "kge.model", "kge.model.embedder", "kge_b200.plugin"])
    config.set("model", "b200_complex")
    config._import("b200_complex")
    config.set("dataset.name", "synthetic")
    config.set("dataset.num_entities", E)
    config.set("dataset.num_relations", R)
    config.set("dataset.pickle", False)
    config.set("job.device", "cuda")
    config.set("job.type", "train")
    config.set("train.type", "negative_sampling")
    config.set("train.loss", "kl")
    config.set("train.batch_size", BATCH)
    config.set("train.num_workers", 0)
    config.set("negative_sampling.class_name", "B200TrainingJobNegativeSampling")
    config.set_all({"lookup_embedder.dim": D, "negative_sampling.num_samples.s": K,
                    "negative_sampling.num_samples.o": K, "negative_sampling.filtering.s": True,
                    "negative_sampling.filtering.o": True, "negative_sampling.filtering.implementation": "fast",
                    "user.b200_device_sampling": device_sampling})
    ds = Dataset(config, None)
    ds._triples = {"train": split}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables("complex", E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job.epoch = 1
    job._prepare()
    assert job._device_sampling == device_sampling
    return job


def time_batch(job, idx):
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    batch = job._get_collate_fun()(idx)
    res = job._process_batch(0, batch)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, res.avg_loss


def kernel_ms(job, tri):
    """Time of the sampling kernels of one batch (S and O), CUDA events over 100 launches."""
    from kge_b200 import engine

    sm = job._sampler
    t = tri.cuda()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rep in range(2):
        torch.cuda.synchronize()
        a.record()
        for i in range(100):
            for slot in (0, 2):
                engine.sample_uniform_filtered(len(t), K, int(sm.vocabulary_size[slot]), 5, (i << 2) | slot, t, slot,
                                               job._filter_index[slot])
        b.record()
        torch.cuda.synchronize()
    return a.elapsed_time(b) / 100


def replaced_fraction(job, tri):
    """Fraction of the draws of both slots whose first id was a positive, for one mirror draw over `tri`."""
    import ns_filter_oracle as nfo

    sm = job._sampler
    hit = total = 0
    for slot in (0, 2):
        ix = job._filter_index[slot]
        _, rep = nfo.sample_uniform_filtered(len(tri), K, int(sm.vocabulary_size[slot]), 5, slot, tri.numpy(), slot,
                                             ix.keys.cpu().numpy(), ix.offsets.cpu().numpy(), ix.values.cpu().numpy(),
                                             return_replaced=True)
        hit += int(rep.sum())
        total += rep.size
    return hit / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    name, power = card()
    rows = []
    for shape, E, R, N in SHAPES:
        split = zipf_split(E, R, N)
        jobs = {"host": make_job(E, R, split, False), "device": make_job(E, R, split, True)}
        idx = torch.randperm(N, generator=torch.Generator().manual_seed(1))[:BATCH].tolist()
        times = {arm: [] for arm in jobs}
        losses = {}
        for rep in range(args.warmup + args.reps):
            for arm, job in jobs.items():                   # alternate the two routes
                ms, loss = time_batch(job, idx)
                losses[arm] = loss
                if rep >= args.warmup:
                    times[arm].append(ms)
        med = {arm: statistics.median(t) for arm, t in times.items()}
        tri = split[idx].long()
        dev = jobs["device"]
        row = {"shape": shape, "E": E, "R": R, "triples": N, "batch": BATCH, "K": K, "D": D, "model": "complex",
               "loss": "kl", **{f"{arm}_ms": round(v, 3) for arm, v in med.items()},
               "speedup": round(med["host"] / med["device"], 2),
               "sampler_kernels_ms": round(kernel_ms(dev, tri), 4),
               "replaced_fraction": replaced_fraction(dev, tri),
               "max_positives_per_key": {s: dev._filter_index[s].max_count for s in (0, 2)},
               "loss_host": losses["host"], "loss_device": losses["device"],
               **{f"{arm}_ms_all": [round(t, 3) for t in v] for arm, v in times.items()}}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del jobs, dev
        torch.cuda.empty_cache()
    print(json.dumps({"card": name, "power_limit_w": power}))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power, "train_batch": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
