"""A/B timing of the headline benchmark between two source trees, on one GPU, in one run.

    python scripts/ab_bench.py TREE_A TREE_B [--rounds 5] [--steps 200] [--out DIR]

Both trees must already be built.  The script alternates `bench.py --gpus 1 --steps S --warmup 5 --no-configs
--dump-outputs ...` between them (A, B, A, B, ...) so that clock and neighbour noise hits both alike, prints the card,
its power limit and SM clocks, the median / min / max of `value`, `roofline.kernel_ms` and `e2e.value` per tree, and
compares the last outputs of the two trees: the loss to 1e-6 relative, the sampled score block bit for bit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def run_bench(tree, steps, dump):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", "5", "--no-configs",
           "--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed in {tree} (rc={r.returncode}):\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trees", nargs=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None, help="directory for the JSON summary and the two trees' last dumps")
    args = ap.parse_args()
    import numpy as np

    trees = [os.path.abspath(t) for t in args.trees]
    out = os.path.abspath(args.out or tempfile.mkdtemp(prefix="ab_bench_"))
    os.makedirs(out, exist_ok=True)
    dumps = [os.path.join(out, f"dump_{i}") for i in range(2)]
    res = {t: {"value": [], "kernel_ms": [], "e2e": []} for t in trees}
    cards = [card()]
    for r in range(args.rounds):
        for t, d in zip(trees, dumps):
            line = run_bench(t, args.steps, d)
            res[t]["value"].append(line["value"])
            res[t]["kernel_ms"].append(line["roofline"]["kernel_ms"])
            res[t]["e2e"].append(line["e2e"]["value"])
            print(json.dumps({"round": r, "tree": t, "value": line["value"], "kernel_ms": line["roofline"]["kernel_ms"],
                              "e2e": line["e2e"]["value"]}), flush=True)
    cards.append(card())
    summary = {"card (name, power limit, SM clock, max SM clock) before / after": cards, "steps": args.steps}
    for t in trees:
        summary[t] = {k: stats(v) for k, v in res[t].items()}
    a, b = trees
    summary["value_ratio_b_over_a"] = summary[b]["value"]["median"] / summary[a]["value"]["median"]
    summary["value_ranges_overlap"] = not (summary[b]["value"]["min"] > summary[a]["value"]["max"] or
                                           summary[a]["value"]["min"] > summary[b]["value"]["max"])
    la, lb = (float(np.load(os.path.join(d, "loss.npy"))[0]) for d in dumps)
    sa, sb = (np.load(os.path.join(d, "scores_sp_po_sample.npy")) for d in dumps)
    diff = np.abs(sa.astype(np.float64) - sb.astype(np.float64))
    summary["outputs"] = {
        "loss": [la, lb], "loss_rel_diff": abs(la - lb) / max(abs(la), 1e-30),
        "scores_bit_identical": bool(np.array_equal(sa.view(np.uint32), sb.view(np.uint32))),
        "scores_max_abs_diff_over_rms": float(diff.max() / np.sqrt(np.mean(sa.astype(np.float64) ** 2))),
        "scores_elements_differing": int((sa.view(np.uint32) != sb.view(np.uint32)).sum()),
    }
    text = json.dumps(summary, indent=1)
    print(text, flush=True)
    with open(os.path.join(out, "ab_summary.json"), "w") as fh:
        fh.write(text + "\n")


if __name__ == "__main__":
    main()
