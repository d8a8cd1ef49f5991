"""Time one training sub-batch (forward + backward, no optimizer step) of a reciprocal-relations model at bench.py's
1vsAll shape (ComplEx, d=512, E=14,541, R=237 so 474 relation rows, n=1024) over three routes that alternate within one
run:

  (a) native   reciprocal_relations_model over b200_complex with the B200 job class: the reciprocal fused step
               (1vsAll) or the sp_ fold of (o, p + R) for the _po query type (KvsAll)
  (b) today    the same model with the unmodified job: the reference's step (embed_all() copies, dense scores,
               scorer-level forward, recompute backward) — the route this configuration took before
  (c) plain    b200_complex (no reciprocal relations) with the B200 job class: the non-reciprocal fused step

for 1vsAll (bce) and KvsAll (kl), each without dropout and with entity / relation dropout 0.4 / 0.2.  CUDA events
around job._process_batch with a synchronise; median of --reps after --warmup rounds.

    python scripts/reciprocal_train_bench.py [--reps 7] [--warmup 2] [--json OUT]

Needs the reference installed (oracle/install_ref.sh) and an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from dropout_train_bench import time_batch  # noqa: E402
from ns_train_bench import card  # noqa: E402

E, R, D, N = 14541, 237, 512, 1024


def make_job(train_type, loss, job_class, reciprocal, p_ent, p_rel):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="reciprocal_bench_")
    config.set("console.quiet", True)
    config.set("modules", ["kge.job", "kge.model", "kge.model.embedder", "kge_b200.plugin"])
    if reciprocal:
        config.set("model", "reciprocal_relations_model")
        config._import("reciprocal_relations_model")
        config._import("b200_complex")
        config.set("reciprocal_relations_model.base_model.type", "b200_complex")
    else:
        config.set("model", "b200_complex")
        config._import("b200_complex")
    config.set("dataset.name", "synthetic")
    config.set("dataset.num_entities", E)
    config.set("dataset.num_relations", R)
    config.set("dataset.pickle", False)
    config.set("job.device", "cuda")
    config.set("job.type", "train")
    config.set("train.type", train_type)
    config.set("train.loss", loss)
    config.set("train.batch_size", N)
    config.set("train.num_workers", 0)
    if job_class:
        config.set(f"{train_type}.class_name", job_class)
    config.set_all({"lookup_embedder.dim": D, "b200_complex.entity_embedder.dropout": p_ent,
                    "b200_complex.relation_embedder.dropout": p_rel})
    ds = Dataset(config, None)
    ds._triples = {"train": synthetic.make_triples(E, R, 4 * N, seed=99).int()}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables("complex", E, 2 * R if reciprocal else R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job._prepare()
    job.model.train()
    return job


def bench(train_type, loss, cls, p_ent, p_rel, reps, warmup):
    jobs = {"native": make_job(train_type, loss, cls, True, p_ent, p_rel),
            "today": make_job(train_type, loss, None, True, p_ent, p_rel),
            "plain": make_job(train_type, loss, cls, False, p_ent, p_rel)}
    batch = next(iter(jobs["native"].loader))
    times = {k: [] for k in jobs}
    values = {}
    for rep in range(warmup + reps):
        for arm, job in jobs.items():                     # alternate the routes
            ms, val = time_batch(job, batch, rep)
            values[arm] = val
            if rep >= warmup:
                times[arm].append(ms)
    med = {k: statistics.median(v) for k, v in times.items()}
    row = {"train_type": train_type, "model": "complex", "loss": loss, "E": E, "R": R, "D": D, "n": N,
           "p_ent": p_ent, "p_rel": p_rel,
           **{f"{k}_ms": round(v, 3) for k, v in med.items()},
           **{f"{k}_ms_all": [round(t, 3) for t in v] for k, v in times.items()},
           "today_over_native": round(med["today"] / med["native"], 2),
           "native_over_plain": round(med["native"] / med["plain"], 2),
           **{f"avg_loss_{k}": v for k, v in values.items()}}
    del jobs
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    name, power = card()
    rows = []
    for train_type, loss, cls in (("1vsAll", "bce", "B200TrainingJob1vsAll"), ("KvsAll", "kl", "B200TrainingJobKvsAll")):
        for p_ent, p_rel in ((0.0, 0.0), (0.4, 0.2)):
            rows.append(bench(train_type, loss, cls, p_ent, p_rel, args.reps, args.warmup))
            print(json.dumps(rows[-1]), flush=True)
    print(json.dumps({"card": name, "power_limit_w": power}))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
