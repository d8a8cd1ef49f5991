"""Time one KvsAll training sub-batch (forward + backward of both query types, no optimizer step) of TransE L1 and
RotatE L1 at the FB15k-237 shape (E=14,541, R=237, d=512, a seeded train split of 272,115 triples from
kge_b200.synthetic.make_triples, 1024 sp_ and 1024 _po queries), over two arms of B200TrainingJobKvsAll that
alternate within one run:

  (a) native     the CSR-label route (forced on in every row): fused score + loss forward, CUDA-core CSR-label
                 backward
  (b) fallback   the same job with only that route disabled (the model's b200_kvsall_native_backward_ok() returns
                 False), i.e. what such a configuration ran before and, without dropout, still runs: the reference's _process_subbatch on the plugin
                 model with dense [n, E] labels, scores and dL/dscores.  Without dropout the tables are read in place
                 and dL/dscores goes to the native dense backward (b200kge_score_1vsN_backward: the same row-gradient
                 passes); with dropout the reference embedders run and the backward recomputes through the reference's
                 torch expression.

Settings: kl with label smoothing 0 and 0.1, each without dropout and with entity / relation dropout 0.4 / 0.2.  CUDA
events around job._process_batch with a synchronise; median of --reps after --warmup rounds; both arms' avg_loss and
their relative difference (without dropout; with dropout the arms draw different masks, the native route from its
Philox key and the reference embedders from torch's generator).  An arm that runs out of device memory is reported as
such.  The card's name and power limit are read in the same run.

    python scripts/kvsall_distance_train_bench.py [--reps 7] [--warmup 2] [--json OUT]

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

E, R, D, N_TRAIN, N_PER_TYPE = 14541, 237, 512, 272115, 1024


def make_job(model, eps, p_ent, p_rel, triples):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    name = "b200_" + model
    config = Config()
    config.folder = tempfile.mkdtemp(prefix="kvsall_distance_bench_")
    config.set("console.quiet", True)
    config.set("modules", ["kge.job", "kge.model", "kge.model.embedder", "kge_b200.plugin"])
    config.set("model", name)
    config._import(name)
    config.set("dataset.name", "synthetic")
    config.set("dataset.num_entities", E)
    config.set("dataset.num_relations", R)
    config.set("dataset.pickle", False)
    config.set("job.device", "cuda")
    config.set("job.type", "train")
    config.set("train.type", "KvsAll")
    config.set("train.loss", "kl")
    config.set("train.batch_size", 2 * N_PER_TYPE)
    config.set("train.num_workers", 0)
    config.set("KvsAll.class_name", "B200TrainingJobKvsAll")
    config.set_all({"lookup_embedder.dim": D, "KvsAll.label_smoothing": eps, f"{name}.l_norm": 1.0,
                    f"{name}.entity_embedder.dropout": p_ent, f"{name}.relation_embedder.dropout": p_rel})
    ds = Dataset(config, None)
    ds._triples = {"train": triples}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables(model, E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job._prepare()
    job.model.train()
    return job


def make_batch(job):
    """N_PER_TYPE seeded queries of each of the sp_ and _po types through the job's own collate."""
    g = torch.Generator().manual_seed(5)
    lo = 0
    idx = []
    for hi in job.query_last_example:
        idx += (lo + torch.randperm(hi - lo, generator=g)[:N_PER_TYPE]).tolist()
        lo = hi
    return job._get_collate_fun()(idx)


def time_batch(job, batch, batch_index):
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = job._process_batch(batch_index, batch)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), res.avg_loss


def bench(model, eps, p_ent, p_rel, triples, reps, warmup):
    from kge_b200 import engine

    jobs = {arm: make_job(model, eps, p_ent, p_rel, triples) for arm in ("native", "fallback")}
    # the job itself takes the CSR-label route for these models under dropout only (the dropout-free rows show why)
    jobs["native"].model.b200_kvsall_native_backward_ok = lambda dropout=False: True
    jobs["fallback"].model.b200_kvsall_native_backward_ok = lambda dropout=False: False
    batch = make_batch(jobs["native"])
    calls = []
    orig = engine.score_1vsN_loss_csr_backward
    engine.score_1vsN_loss_csr_backward = lambda *a, **kw: calls.append(1) or orig(*a, **kw)
    times = {k: [] for k in jobs}
    values, failed = {}, {}
    try:
        for rep in range(warmup + reps):
            for arm, job in jobs.items():                 # alternate the arms; the same masks key per rep
                if arm in failed:
                    continue
                n0 = len(calls)
                try:
                    ms, val = time_batch(job, batch, rep)
                except torch.cuda.OutOfMemoryError:
                    failed[arm] = "CUDA out of memory"
                    job.model.zero_grad(set_to_none=True)
                    torch.cuda.empty_cache()
                    continue
                assert (len(calls) > n0) == (arm == "native"), arm
                values[arm] = val
                if rep >= warmup:
                    times[arm].append(ms)
    finally:
        engine.score_1vsN_loss_csr_backward = orig
    med = {k: (statistics.median(v) if k not in failed else None) for k, v in times.items()}
    counts = torch.bincount(batch["query_type_indexes"], minlength=2).tolist()
    row = {"model": model, "l_norm": 1.0, "loss": "kl", "label_smoothing": eps, "p_ent": p_ent, "p_rel": p_rel,
           "E": E, "D": D, "queries_sp": counts[0], "queries_po": counts[1],
           **{f"{k}_ms": (round(v, 3) if v is not None else failed[k]) for k, v in med.items()},
           **{f"{k}_ms_all": [round(t, 3) for t in v] for k, v in times.items()},
           **{f"avg_loss_{k}": v for k, v in values.items()}}
    if not failed:
        row["fallback_over_native"] = round(med["fallback"] / med["native"], 2)
        row["avg_loss_rel_diff"] = abs(values["native"] - values["fallback"]) / abs(values["fallback"])
    del jobs
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from kge_b200 import synthetic

    torch.manual_seed(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit_w": power}), flush=True)
    triples = synthetic.make_triples(E, R, N_TRAIN, seed=237).int()
    rows = []
    for model in ("transe", "rotate"):
        for eps in (0.0, 0.1):
            for p_ent, p_rel in ((0.0, 0.0), (0.4, 0.2)):
                rows.append(bench(model, eps, p_ent, p_rel, triples, args.reps, args.warmup))
                print(json.dumps(rows[-1]), flush=True)
    _, power2 = card()
    out = {"card": name, "power_limit_w": power, "power_limit_w_after": power2, "rows": rows}
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
