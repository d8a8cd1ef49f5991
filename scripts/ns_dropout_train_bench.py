"""Time one negative-sampling training batch with embedding dropout (forward + backward of the S and O slots, no
optimizer step), three routes of B200TrainingJobNegativeSampling alternated in one process:

  (a) dropout   user.b200_ns_dropout: true — masked scores (b200kge_ns_score_dropout) -> row-loss kernel -> masked
                backward (b200kge_ns_backward with the key)
  (b) fallback  the same job without the option: the reference's _process_subbatch (reference embedders, torch dropout,
                eager scoring, autograd)
  (c) nodrop    the native NS step with dropout 0 (what the batch costs without dropout)

at two shapes: K = 30 (`auto` resolves to `triple`) and K = 1000 (`batch`).  Median of --reps after --warmup, CUDA events
with a synchronise.  Once per configuration a parity line compares the loss of (a) with the reference step whose
embedders apply the masks of engine.dropout_mask under the same key (tests/ns_dropout_oracle.py).

    python scripts/ns_dropout_train_bench.py [--reps 7] [--batch 512] [--json OUT]

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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from ns_train_bench import card  # noqa: E402

E, R, D = 40943, 11, 512
P_ENT, P_REL = 0.4, 0.2
MODELS = ("complex", "rotate")
SHAPES = ((30, "triple"), (1000, "batch"))


def make_job(model, K, batch):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="ns_dropout_bench_")
    config.set("console.quiet", True)
    config.set("modules", ["kge.job", "kge.model", "kge.model.embedder", "kge_b200.plugin"])
    config.set("model", "b200_" + model)
    config._import("b200_" + model)
    config.set("dataset.name", "synthetic")
    config.set("dataset.num_entities", E)
    config.set("dataset.num_relations", R)
    config.set("dataset.pickle", False)
    config.set("job.device", "cuda")
    config.set("job.type", "train")
    config.set("train.type", "negative_sampling")
    config.set("train.loss", "kl")
    config.set("train.batch_size", batch)
    config.set("train.num_workers", 0)
    config.set("negative_sampling.class_name", "B200TrainingJobNegativeSampling")
    config.set_all({"lookup_embedder.dim": D, "negative_sampling.num_samples.s": K,
                    "negative_sampling.num_samples.o": K, "negative_sampling.implementation": "auto",
                    f"b200_{model}.entity_embedder.dropout": P_ENT, f"b200_{model}.relation_embedder.dropout": P_REL,
                    "user.b200_ns_dropout": True})
    ds = Dataset(config, None)
    ds._triples = {"train": synthetic.make_triples(E, R, 4 * batch, seed=99).int()}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables(model, E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job.epoch = 1
    job._prepare()
    return job


def set_arm(job, arm):
    m = job.model
    job.config.set("user.b200_ns_dropout", arm == "dropout")
    m.get_s_embedder().dropout.p = 0.0 if arm == "nodrop" else P_ENT
    m.get_p_embedder().dropout.p = 0.0 if arm == "nodrop" else P_REL
    m.__dict__.pop("_b200_fusable_cache", None)          # the rates changed


def time_batch(job, batch):
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = job._process_batch(0, batch)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), res.avg_loss


def parity(job, batch):
    """Loss of route (a) and of the reference step drawing engine.dropout_mask's masks under the same key."""
    import ns_dropout_oracle as nso
    from kge_b200 import engine

    set_arm(job, "dropout")
    job._b200_drop_pos = None
    native = job._process_batch(0, batch).avg_loss

    def mask_rows(p, key, strm, rows, dim):
        rows = torch.as_tensor(rows).long().reshape(-1)
        lo, hi = int(rows.min()), int(rows.max()) + 1
        m = engine.dropout_mask(p, key.seed, key.call, strm, hi - lo, dim, lo)
        return m[(rows - lo).to(m.device)].bool()

    nso.mask_rows = mask_rows
    set_arm(job, "fallback")
    nso.patch_reference_ns_job(job, P_ENT, P_REL)
    ref = job._process_batch(0, batch).avg_loss
    return native, ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    name, power = card()
    rows = []
    for model in MODELS:
        for K, impl in SHAPES:
            job = make_job(model, K, args.batch)
            assert job._implementation == impl, (job._implementation, impl)
            batch = next(iter(job.loader))
            times = {"dropout": [], "fallback": [], "nodrop": []}
            oom = set()
            for rep in range(args.warmup + args.reps):
                for arm in times:                              # alternate the three routes
                    if arm in oom:
                        continue
                    set_arm(job, arm)
                    try:
                        ms, _ = time_batch(job, batch)
                    except RuntimeError as e:                  # the reference's batch route of RotatE at K = 1000
                        if "out of memory" not in str(e):
                            raise
                        oom.add(arm)
                        job.model.zero_grad(set_to_none=True)
                        torch.cuda.empty_cache()
                        continue
                    if rep >= args.warmup:
                        times[arm].append(ms)
            med = {arm: (statistics.median(t) if arm not in oom else None) for arm, t in times.items()}
            native, ref = parity(job, batch) if "fallback" not in oom else (None, None)
            row = {"model": model, "K": K, "implementation": impl, "D": D, "E": E, "batch": args.batch,
                   "p_ent": P_ENT, "p_rel": P_REL, "loss": "kl",
                   **{f"{arm}_ms": (round(v, 3) if v is not None else "out of memory") for arm, v in med.items()},
                   "speedup_vs_fallback": round(med["fallback"] / med["dropout"], 2) if med["fallback"] else None,
                   "parity_loss_native": native, "parity_loss_ref": ref,
                   "parity_rel": abs(native - ref) / max(abs(ref), 1e-30) if ref is not None else None,
                   **{f"{arm}_ms_all": [round(t, 3) for t in v] for arm, v in times.items()}}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del job
            torch.cuda.empty_cache()
    print(json.dumps({"card": name, "power_limit_w": power}))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power, "train_batch": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
