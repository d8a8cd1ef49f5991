"""Time frequency negative sampling on the device against uniform device sampling, in one process, arms alternated:

  kernels  the sampling entries alone for one batch (S and O slots, K = 1000, 512 triples): b200kge_sample_frequency
           against b200kge_sample_uniform, and b200kge_sample_frequency_filtered against b200kge_sample_uniform_filtered
           on the same triples and filter index; CUDA events over 20 launches per sample
  train    one negative-sampling training batch of B200TrainingJobNegativeSampling with user.b200_device_sampling,
           forward + backward of the S and O slots (no optimizer step), filtering.s and .o on, including the collate;
           the same job runs both arms: its frequency tables are switched off for the uniform arm

Triples come from a seeded split whose subjects and objects follow Zipf(1.0) (as scripts/ns_filter_bench.py), at a
WN18RR shape (40,943 entities, 11 relations, 86,835 triples) and a Wikidata5M-sized entity vocabulary (4.8M entities,
822 relations, 5M triples; the frequency CDF is then 38 MB).  ComplEx, kl, d = 512, batch 512.  Median of --reps after
--warmup.  The card's name and power limit are read in the same run.

There is no host arm: the reference's frequency sampler (KgeFrequencySampler) cannot be constructed on current torch,
which no longer has torch._multinomial_alias_setup.

    python scripts/ns_frequency_bench.py [--reps 7] [--shapes WN18RR,Wikidata5M] [--json OUT]

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
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from ns_filter_bench import zipf_split  # noqa: E402
from ns_train_bench import card  # noqa: E402

SHAPES = {"WN18RR": (40943, 11, 86835), "Wikidata5M": (4_800_000, 822, 5_000_000)}
D, K, BATCH, LAUNCHES = 512, 1000, 512, 20
NO_HOST_ARM = ("no host arm: the reference's KgeFrequencySampler cannot be constructed on this torch "
               "(torch._multinomial_alias_setup does not exist)")


def make_job(E, R, split):
    from kge_b200 import hostenv

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="ns_frequency_bench_")
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
                    "negative_sampling.filtering.o": True, "negative_sampling.sampling_type": "frequency",
                    "user.b200_device_sampling": True})
    ds = Dataset(config, None)
    ds._triples = {"train": split}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    job.epoch = 1
    job._prepare()
    assert job._device_sampling and sorted(job._frequency) == [0, 2] and sorted(job._filter_index) == [0, 2]
    return job


def time_batch(job, idx, frequency, tables):
    job._frequency = tables if frequency else {}
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    batch = job._get_collate_fun()(idx)
    res = job._process_batch(0, batch)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, res.avg_loss


def kernel_arms(job, tables, tri):
    """{arm: callable drawing both slots of one batch} on the job's tables and filter indexes."""
    from kge_b200 import engine

    t = tri.cuda()
    ix = job._filter_index
    V = {s: tables[s].vocab for s in (0, 2)}
    return {
        "uniform": lambda i: [engine.sample_uniform(len(t), K, V[s], 5, (i << 2) | s, "cuda") for s in (0, 2)],
        "frequency": lambda i: [engine.sample_frequency(len(t), K, tables[s], 5, (i << 2) | s) for s in (0, 2)],
        "uniform_filtered": lambda i: [engine.sample_uniform_filtered(len(t), K, V[s], 5, (i << 2) | s, t, s, ix[s])
                                       for s in (0, 2)],
        "frequency_filtered": lambda i: [engine.sample_frequency_filtered(len(t), K, tables[s], 5, (i << 2) | s, t, s,
                                                                          ix[s]) for s in (0, 2)],
    }


def kernel_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(LAUNCHES):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / LAUNCHES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit_w": power, "note": NO_HOST_ARM}), flush=True)
    rows = []
    for shape in args.shapes.split(","):
        E, R, N = SHAPES[shape]
        split = zipf_split(E, R, N)
        job = make_job(E, R, split)
        tables = dict(job._frequency)
        idx = torch.randperm(N, generator=torch.Generator().manual_seed(1))[:BATCH].tolist()
        tri = split[idx].long()
        arms = kernel_arms(job, tables, tri)
        kt = {arm: [] for arm in arms}
        tt = {arm: [] for arm in ("uniform", "frequency")}
        losses = {}
        for rep in range(args.warmup + args.reps):
            for arm, fn in arms.items():                      # alternate the arms
                ms = kernel_ms(fn)
                if rep >= args.warmup:
                    kt[arm].append(ms)
            for arm in tt:
                ms, losses[arm] = time_batch(job, idx, arm == "frequency", tables)
                if rep >= args.warmup:
                    tt[arm].append(ms)
        job._frequency = tables
        kmed = {arm: statistics.median(v) for arm, v in kt.items()}
        tmed = {arm: statistics.median(v) for arm, v in tt.items()}
        row = {"shape": shape, "E": E, "R": R, "triples": N, "batch": BATCH, "K": K, "D": D, "model": "complex",
               "loss": "kl", "filtering": "s,o",
               **{f"kernels_{arm}_ms": round(v, 4) for arm, v in kmed.items()},
               **{f"train_{arm}_ms": round(v, 3) for arm, v in tmed.items()},
               "train_frequency_over_uniform": round(tmed["frequency"] / tmed["uniform"], 3),
               "frequency_filtered_kernels_share_of_step": round(kmed["frequency_filtered"] / tmed["frequency"], 4),
               "loss_uniform": losses["uniform"], "loss_frequency": losses["frequency"],
               **{f"train_{arm}_ms_all": [round(t, 3) for t in v] for arm, v in tt.items()}}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del job, arms, tables
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power, "note": NO_HOST_ARM, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
