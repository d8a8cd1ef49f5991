"""Time one validation epoch of LibKGE's entity-ranking evaluation on a plugin model, two arms alternating in one run:

  (a) B200EntityRankingJob     one b200kge_rank_sp_po_eval call per batch (+ score_sp / score_po for the true scores)
  (b) EntityRankingJob         the unmodified job on the same model: score_sp_po per chunk, dense label matrices and
                               the torch ranking passes

at two shapes:

  fb15k237    ComplEx d=512, E=14,541, R=237, a 272,115-triple synthetic train split as filter, 17,535 eval triples
  wikidata5m  TransE L1 d=512, E=4,800,000, R=828, a 2,000,000-triple synthetic train split as filter, --wd-eval eval
              triples (default 2,000); arm (b) with entity_ranking.chunk_size --wd-chunk (default 200,000: one chunk's
              scores and labels are [100, 400,000] floats, 160 MB each)

eval.batch_size 100, filter_with_test on.  Host clock around valid_job._run() ending in a device synchronise, median of
--reps per arm.  Also checks that both arms' metrics are equal, and times the ranking entry of one batch with CUDA
events (the whole call: folds, operand split and the scorer) and the scorer kernel alone.

    python scripts/eval_bench.py [--shapes fb15k237,wikidata5m] [--reps 5] [--json OUT]

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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from ns_train_bench import card  # noqa: E402

SHAPES = {
    "fb15k237": dict(model="complex", E=14541, R=237, n_train=272115, n_eval=17535, chunk=-1),
    "wikidata5m": dict(model="transe", E=4_800_000, R=828, n_train=2_000_000, n_eval=2000, chunk=200_000),
}
METRICS = [k + s for s in ("", "_filtered", "_filtered_with_test")
           for k in ("mean_rank", "mean_reciprocal_rank", "hits_at_1", "hits_at_3", "hits_at_10")]


def make_jobs(shape):
    from kge_b200 import hostenv, synthetic

    hostenv.import_kge()
    from kge import Config, Dataset
    from kge.job import EvaluationJob, TrainingJob

    name = "b200_" + shape["model"]
    E, R, D = shape["E"], shape["R"], 512
    config = Config()
    config.folder = tempfile.mkdtemp(prefix="eval_bench_")
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
    config.set("train.type", "1vsAll")
    config.set("eval.batch_size", 100)
    config.set("eval.num_workers", 0)
    config.set("entity_ranking.filter_with_test", True)
    config.set("entity_ranking.chunk_size", shape["chunk"])
    config.set("entity_ranking.class_name", "B200EntityRankingJob")
    config.set_all({"lookup_embedder.dim": D})
    if shape["model"] == "transe":
        config.set(f"{name}.l_norm", 1.0)
    ds = Dataset(config, None)
    ds._triples = {"train": synthetic.make_triples(E, R, shape["n_train"], seed=5).int(),
                   "valid": synthetic.make_triples(E, R, shape["n_eval"], seed=6).int(),
                   "test": synthetic.make_triples(E, R, shape["n_eval"], seed=7).int()}
    ds._meta = {"entity_ids": [str(i) for i in range(E)], "relation_ids": [str(i) for i in range(R)]}
    job = TrainingJob.create(config, ds)
    ent, rel = synthetic.make_tables(shape["model"], E, R, D, sigma=0.1)
    with torch.no_grad():
        job.model.get_s_embedder()._embeddings.weight.copy_(ent)
        job.model.get_p_embedder()._embeddings.weight.copy_(rel)
    fused = job.valid_job
    conf = fused.config.clone()
    conf.set("entity_ranking.class_name", "EntityRankingJob")
    ref = EvaluationJob.create(conf, ds, parent_job=job, model=job.model)
    for ev in (fused, ref):
        ev._prepare()
    assert type(fused).__name__ == "B200EntityRankingJob" and fused._b200_route is not None
    assert type(ref).__name__ == "EntityRankingJob"
    return fused, ref


def run_epoch(ev):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = ev._run()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def entry_time(ev, reps=20):
    """(ms per ranking call, ms of its scorer kernel) for the first batch, CUDA events."""
    from kge_b200 import engine

    batch, filt, test, own = next(iter(ev.loader))
    dev = "cuda"
    batch = batch.to(dev)
    s, p, o = batch[:, 0], batch[:, 1], batch[:, 2]
    filt = tuple(t.to(dev) for t in filt)
    test = tuple(t.to(dev) for t in test) or None
    own = own.to(dev)
    model, recip = ev._b200_route
    with torch.no_grad():
        ev.model.eval()
        true2n = ev._b200_true_scores(s, p, o)
        call = lambda: model.rank_eval(s, p, o, true2n, filt, test, ev.tie_rtol, ev.tie_atol, reciprocal=recip,  # noqa
                                       own_col=own)
        call()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call()
        b.record()
        torch.cuda.synchronize()
        engine.profile_enable(True)
        call()
        scorer = engine.profile_last_ms()
        engine.profile_enable(False)
    return a.elapsed_time(b) / reps, scorer


def bench(shape_name, reps):
    shape = SHAPES[shape_name]
    fused, ref = make_jobs(shape)
    run_epoch(fused)                         # warm-up: module load, workspaces, index building
    run_epoch(ref)
    times = {"b200": [], "reference": []}
    outs = {}
    for _ in range(reps):
        for tag, ev in (("b200", fused), ("reference", ref)):
            dt, out = run_epoch(ev)
            times[tag].append(dt)
            outs[tag] = out
    diff = {k: (outs["b200"][k], outs["reference"][k]) for k in METRICS if outs["b200"][k] != outs["reference"][k]}
    call_ms, scorer_ms = entry_time(fused)
    res = {"shape": shape_name, **{k: v for k, v in shape.items()}, "batch_size": 100, "reps": reps,
           "b200_s": statistics.median(times["b200"]), "reference_s": statistics.median(times["reference"]),
           "b200_all_s": times["b200"], "reference_all_s": times["reference"],
           "metrics_equal": not diff, "metric_diffs": diff,
           "mrr_filtered": outs["b200"]["mean_reciprocal_rank_filtered"],
           "entry_call_ms": call_ms, "entry_scorer_ms": scorer_ms}
    res["speedup"] = res["reference_s"] / res["b200_s"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="fb15k237,wikidata5m")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--wd-eval", type=int, default=2000)
    ap.add_argument("--wd-chunk", type=int, default=200_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    SHAPES["wikidata5m"].update(n_eval=args.wd_eval, chunk=args.wd_chunk)
    name, power = card()
    print(json.dumps({"card": name, "power_limit_w": power}), flush=True)
    results = []
    for sh in args.shapes.split(","):
        r = bench(sh, args.reps)
        results.append(r)
        print(json.dumps(r), flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power, "results": results}, fh, indent=1)


if __name__ == "__main__":
    main()
