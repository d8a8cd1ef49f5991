"""Time one training sub-batch (forward + backward, no optimizer step) with embedding dropout at bench.py's 1vsAll shape
(ComplEx, d=512, E=14,541, R=237, n=1024, bce; entity_embedder.dropout 0.4, relation_embedder.dropout 0.2), over three
routes that alternate within one run:

  (a) native   B200TrainingJob1vsAll with dropout: the dropout entry points (masks drawn on the device)
  (b) today    the unmodified TrainingJob1vsAll on b200_complex with the same dropout (reference embedders, embed_all()
               copies, scorer-level forward, recompute backward) — the route this configuration took before
  (c) p=0      B200TrainingJob1vsAll without dropout: the fused step

plus the same three routes for KvsAll (ComplEx, kl).  CUDA events around job._process_batch with a synchronise; median
of --reps after --warmup rounds.  Also prints a rough estimate of the extra HBM traffic of route (a)'s materialised
table copies from the data-sheet bandwidth.

    python scripts/dropout_train_bench.py [--reps 7] [--warmup 2] [--json OUT]

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

from ns_train_bench import card  # noqa: E402

E, R, D, N = 14541, 237, 512, 1024
P_ENT, P_REL = 0.4, 0.2
PEAK_BW = 3.35e12          # H100 SXM HBM3 data-sheet bandwidth, bytes/s


def make_job(train_type, loss, job_class, p_ent, p_rel):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="dropout_bench_")
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
    ent, rel = synthetic.make_tables("complex", E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job._prepare()
    job.model.train()
    return job


def time_batch(job, batch, batch_index):
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = job._process_batch(batch_index, batch)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), res.avg_loss


def bench(train_type, loss, cls, reps, warmup):
    jobs = {"native": make_job(train_type, loss, cls, P_ENT, P_REL),
            "today": make_job(train_type, loss, None, P_ENT, P_REL),
            "p0": make_job(train_type, loss, cls, 0.0, 0.0)}
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
    row = {"train_type": train_type, "model": "complex", "loss": loss, "E": E, "D": D, "n": len(batch.get(
        "triples", batch.get("queries"))), "p_ent": P_ENT, "p_rel": P_REL,
        **{f"{k}_ms": round(v, 3) for k, v in med.items()},
        **{f"{k}_ms_all": [round(t, 3) for t in v] for k, v in times.items()},
        "today_over_native": round(med["today"] / med["native"], 2),
        "native_over_p0": round(med["native"] / med["p0"], 2),
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
        rows.append(bench(train_type, loss, cls, args.reps, args.warmup))
        print(json.dumps(rows[-1]), flush=True)
    # rough estimate, not a measurement: bytes the table copies add to a 1vsAll step (per direction: forward gather
    # read + write; backward gather read + write, dT write, masked add reads dT and reads + writes d_ent)
    table = E * D * 4
    extra = 2 * (2 + 2 + 1 + 3) * table
    est = {"estimate": "extra HBM bytes of the materialised table copies per 1vsAll step, at data-sheet bandwidth",
           "bytes": extra, "ms_at_data_sheet_bw": round(extra / PEAK_BW * 1e3, 3)}
    print(json.dumps(est))
    out = {"card": name, "power_limit_w": power, "rows": rows, "table_copy_estimate": est}
    print(json.dumps({"card": name, "power_limit_w": power}))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
