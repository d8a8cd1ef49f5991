"""Time one KvsAll training sub-batch (forward + backward of every query type, no optimizer step) with the query types
sp_ + s_o + _po, ComplEx at the FB15k-237 shape (E=14,541, R=237, d=512, a seeded train split of 272,115 triples from
kge_b200.synthetic.make_triples, 1024 queries per query type), over three arms of B200TrainingJobKvsAll that alternate
within one run:

  (a) so         the s_o route: the s_o rows through b200kge_score_so_loss_csr and its backward, sp_ and _po fused
  (b) fallback   the same job with only the s_o route switched off (the model's b200_kvsall_so_ok() returns False),
                 i.e. what the job ran before for a configuration with s_o: the reference's _process_subbatch for the
                 whole sub-batch (dense labels; without dropout dense scores and the native dense backward, with dropout
                 the reference embedders)
  (c) sp_po      the fused job with the query types sp_ + _po only, for context (its own batch of 2 x 1024 queries)

Settings: kl, without dropout and with entity / relation dropout 0.4 / 0.2.  CUDA events around job._process_batch
with a synchronise; median of --reps after --warmup rounds; the arms' avg_loss (without dropout (a) and (b) compute the
same value; with dropout they draw different masks).  An arm that runs out of device memory is reported as such.  The
card's name and power limit are read in the same run.

    python scripts/kvsall_so_train_bench.py [--reps 7] [--warmup 2] [--json OUT]

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

from kvsall_distance_train_bench import make_batch, time_batch  # noqa: E402
from ns_train_bench import card  # noqa: E402

MODEL, E, R, D, N_TRAIN = "complex", 14541, 237, 512, 272115


def make_job(with_so, p_ent, p_rel, triples):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    name = "b200_" + MODEL
    config = Config()
    config.folder = tempfile.mkdtemp(prefix="kvsall_so_bench_")
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
    config.set("train.batch_size", 3072)
    config.set("train.num_workers", 0)
    config.set("KvsAll.class_name", "B200TrainingJobKvsAll")
    config.set_all({"lookup_embedder.dim": D, "KvsAll.query_types.s_o": with_so,
                    f"{name}.entity_embedder.dropout": p_ent, f"{name}.relation_embedder.dropout": p_rel})
    ds = Dataset(config, None)
    ds._triples = {"train": triples}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables(MODEL, E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job._prepare()
    job.model.train()
    return job


def bench(p_ent, p_rel, triples, reps, warmup):
    from kge_b200 import engine

    jobs = {"so": make_job(True, p_ent, p_rel, triples), "fallback": make_job(True, p_ent, p_rel, triples),
            "sp_po": make_job(False, p_ent, p_rel, triples)}
    jobs["fallback"].model.b200_kvsall_so_ok = lambda: False
    batches = {arm: make_batch(job) for arm, job in jobs.items()}
    calls = []
    orig = engine.score_so_loss_csr_backward
    engine.score_so_loss_csr_backward = lambda *a, **kw: calls.append(1) or orig(*a, **kw)
    times = {k: [] for k in jobs}
    values, failed = {}, {}
    try:
        for rep in range(warmup + reps):
            for arm, job in jobs.items():                 # alternate the arms; the same masks key per rep
                if arm in failed:
                    continue
                n0 = len(calls)
                try:
                    ms, val = time_batch(job, batches[arm], rep)
                except torch.cuda.OutOfMemoryError:
                    failed[arm] = "CUDA out of memory"
                    job.model.zero_grad(set_to_none=True)
                    torch.cuda.empty_cache()
                    continue
                assert (len(calls) > n0) == (arm == "so"), arm
                values[arm] = val
                if rep >= warmup:
                    times[arm].append(ms)
    finally:
        engine.score_so_loss_csr_backward = orig
    med = {k: (statistics.median(v) if k not in failed else None) for k, v in times.items()}
    counts = torch.bincount(batches["so"]["query_type_indexes"], minlength=3).tolist()
    row = {"model": MODEL, "loss": "kl", "p_ent": p_ent, "p_rel": p_rel, "E": E, "R": R, "D": D,
           "queries_per_type": counts,
           **{f"{k}_ms": (round(v, 3) if v is not None else failed[k]) for k, v in med.items()},
           **{f"{k}_ms_all": [round(t, 3) for t in v] for k, v in times.items()},
           **{f"avg_loss_{k}": v for k, v in values.items()}}
    if "so" not in failed and "fallback" not in failed:
        row["fallback_over_so"] = round(med["fallback"] / med["so"], 2)
        row["avg_loss_rel_diff"] = abs(values["so"] - values["fallback"]) / abs(values["fallback"])
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
    for p_ent, p_rel in ((0.0, 0.0), (0.4, 0.2)):
        rows.append(bench(p_ent, p_rel, triples, args.reps, args.warmup))
        print(json.dumps(rows[-1]), flush=True)
    _, power2 = card()
    out = {"card": name, "power_limit_w": power, "power_limit_w_after": power2, "rows": rows}
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
