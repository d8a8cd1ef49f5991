"""Time one negative-sampling training batch (forward + backward of the S and O slots, no optimizer step) with the
losses beyond plain bce: the native route of B200TrainingJobNegativeSampling (ns_score -> row-loss kernel -> G-driven
NS backward) against the route it replaces (the same job with `model.b200_backward = "reference"`: the reference's
_process_subbatch, scores through the plugin, backward by recomputing the reference's dense expression).  The two arms
alternate in one run; CUDA events with a synchronise.  Also times the row-loss kernel alone against its HBM bound.

    python scripts/ns_train_bench.py [--reps 5] [--batch 512] [--json OUT]

Needs the reference installed (oracle/install_ref.sh) and an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

E, R, D, K = 40943, 11, 512, 1000
CONFIGS = [("rotate", "kl"), ("rotate", "bce_self_adversarial"), ("rotate", "margin_ranking"),
           ("complex", "kl"), ("complex", "bce_self_adversarial"), ("complex", "margin_ranking")]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def make_job(model, loss, batch):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import TrainingJob

    config = Config()
    config.folder = tempfile.mkdtemp(prefix="ns_bench_")
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
    config.set("train.loss", loss)
    config.set("train.batch_size", batch)
    config.set("train.num_workers", 0)
    config.set("negative_sampling.class_name", "B200TrainingJobNegativeSampling")
    config.set_all({"lookup_embedder.dim": D, "negative_sampling.num_samples.s": K,
                    "negative_sampling.num_samples.o": K, "negative_sampling.implementation": "triple"})
    ds = Dataset(config, None)
    ds._triples = {"train": synthetic.make_triples(E, R, 4 * batch, seed=99).int()}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables(model, E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    job._prepare()
    return job


def time_batch(job, batch):
    """ms of job._process_batch (forward + backward of every slot), gradients cleared first."""
    job.model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = job._process_batch(0, batch)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), res.avg_loss


def time_loss_kernel(n, m, loss, want_grad, reps=20):
    from kge_b200 import engine

    z = torch.randn((n, m), device="cuda") * 3
    for _ in range(3):
        engine.ns_loss(z, loss, 0.5, 1.0, want_grad=want_grad)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        engine.ns_loss(z, loss, 0.5, 1.0, want_grad=want_grad)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    name, power = card()
    rows = []
    for model, loss in CONFIGS:
        job = make_job(model, loss, args.batch)
        batch = next(iter(job.loader))
        times = {"native": [], "fallback": []}
        values = {}
        for rep in range(args.warmup + args.reps):
            for arm in ("native", "fallback"):              # alternate the two routes
                job.model.b200_backward = "native" if arm == "native" else "reference"
                ms, val = time_batch(job, batch)
                values[arm] = val
                if rep >= args.warmup:
                    times[arm].append(ms)
        nat, fb = statistics.median(times["native"]), statistics.median(times["fallback"])
        row = {"model": model, "loss": loss, "D": D, "E": E, "K": K, "batch": args.batch, "slots": "s,o",
               "native_ms": round(nat, 3), "fallback_ms": round(fb, 3), "speedup": round(fb / nat, 2),
               "native_ms_all": [round(t, 3) for t in times["native"]],
               "fallback_ms_all": [round(t, 3) for t in times["fallback"]],
               "avg_loss_native": values["native"], "avg_loss_fallback": values["fallback"]}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del job
        torch.cuda.empty_cache()
    kernel = []
    peak = 3.35e12        # H100 SXM HBM3 data-sheet bandwidth, bytes/s
    for loss in ("kl", "bce_self_adversarial", "margin_ranking"):
        for n, want_grad in ((args.batch, False), (args.batch, True), (65536, False), (65536, True)):
            m = 1 + K
            ms = time_loss_kernel(n, m, loss, want_grad)
            nbytes = n * m * 4 * (2 if want_grad else 1)
            kernel.append({"loss": loss, "n": n, "m": m, "grad": want_grad, "ms": round(ms, 4),
                           "hbm_bound_ms": round(nbytes / peak * 1e3, 4), "GBps": round(nbytes / ms / 1e6, 1)})
            print(json.dumps(kernel[-1]), flush=True)
    out = {"card": name, "power_limit_w": power, "train_batch": rows, "row_loss_kernel": kernel}
    print(json.dumps({"card": name, "power_limit_w": power}))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
