"""Kernel micro-benchmarks on the GPU box (development aid, not the driver's bench).

Times the dominant kernel of several calls with the library's own CUDA-event brackets
(b200kge_profile_*), after warm-up, with L2 flushed between iterations, and prints one JSON line per
case.  Usage: python scripts/kbench.py [case ...]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from kge_b200 import engine  # noqa: E402
from kge_b200 import synthetic  # noqa: E402
from oracle import kge_oracle as orc  # noqa: E402  (the parity cases use it as the checker)

dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    engine.profile_enable(True)
    ks, ts = [], []
    for i in range(iters):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
        ks.append(engine.profile_last_ms())
    engine.profile_enable(False)
    return sum(ks) / len(ks), min(ks), sum(ts) / len(ts)


def case_1vsall(model, E, R, D, n, prec, epi, l_norm=1.0):
    ent, rel = synthetic.make_tables(model, E, R, D)
    tri = synthetic.make_triples(E, R, n).to(dev)
    ent, rel = ent.to(dev), rel.to(dev)
    s, p, o = tri[:, 0].contiguous(), tri[:, 1].contiguous(), tri[:, 2].contiguous()
    if epi == "store":
        fn = lambda: engine.score_sp_po(model, ent, rel, s, p, o, None, l_norm, prec)
    elif epi == "step":
        ws = engine._workspace(0, n, E, D, False, dev)
        out = torch.zeros((), device=dev)
        fn = lambda: engine.train_1vsall_forward(model, ent, rel, tri, "bce", 0.0, l_norm, prec, out, ws)
    elif epi == "kl":
        ws = engine._workspace(0, n, E, D, False, dev)
        out = torch.zeros((), device=dev)
        fn = lambda: engine.train_1vsall_forward(model, ent, rel, tri, "kl", 0.0, l_norm, prec, out, ws)
    k_avg, k_min, t_avg = timeit(fn)
    pairs = 2.0 * n * E
    print(json.dumps({"case": f"{model} E={E} D={D} n={n} {prec} {epi}", "kernel_ms": round(k_avg, 4),
                      "kernel_ms_min": round(k_min, 4), "call_ms": round(t_avg, 4),
                      "Gpairs_per_s": round(pairs / k_avg / 1e6, 2),
                      "alg_TFLOPs": round(pairs * 2 * D / k_avg / 1e9, 2)}), flush=True)


def case_kvsall(model, E, R, D, n, loss):
    """Fused score_sp + loss with DENSE multi-hot labels (KvsAll, train_KvsAll.py:242-289)."""
    ent, rel = synthetic.make_tables(model, E, R, D, sigma=0.3)
    tri = synthetic.make_triples(E, R, n).to(dev)
    ent, rel = ent.to(dev), rel.to(dev)
    lab = (torch.rand((n, E), device=dev) < 2e-4).float()
    s, p = tri[:, 0].contiguous(), tri[:, 1].contiguous()
    fn = lambda: engine.score_1vsN_loss(model, "sp_", ent, rel, ent, lab, s, p, None, loss)
    k_avg, k_min, t_avg = timeit(fn)
    print(json.dumps({"case": f"kvsall {model} E={E} D={D} n={n} {loss} dense labels", "kernel_ms": round(k_avg, 4),
                      "call_ms": round(t_avg, 4), "label_GB": round(n * E * 4 / 1e9, 3),
                      "label_GBps": round(n * E * 4 / k_avg / 1e6, 1)}), flush=True)


def case_ns(model, E, R, D, n, K):
    ent, rel = synthetic.make_tables(model, E, R, D)
    tri = synthetic.make_triples(E, R, n).to(dev)
    ent, rel = ent.to(dev), rel.to(dev)
    neg = torch.randint(0, E, (n, K), device=dev)
    fn = lambda: engine.ns_score(model, ent, rel, tri, neg, 2, True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for i in range(10):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    t = sum(ts) / len(ts)
    gathered = n * K * D * 4.0
    print(json.dumps({"case": f"ns {model} E={E} D={D} n={n} K={K}", "call_ms": round(t, 4),
                      "Mscores_per_s": round(n * (K + 1) / t / 1e3, 1),
                      "gather_GBps": round(gathered / t / 1e6, 1)}), flush=True)


def case_parity():
    """max|d|/rms of the TC path vs the fp32 SIMT path and vs the fp64 oracle (n=256 sample)."""
    model, E, R, D, n = "complex", 14541, 237, 512, 256
    ent, rel = synthetic.make_tables(model, E, R, D)
    tri = synthetic.make_triples(E, R, n)
    ref = orc.score_sp(model, ent.double(), rel.double(), tri[:, 0], tri[:, 1])
    rms = float(ref.pow(2).mean().sqrt())
    e, r, t = ent.to(dev), rel.to(dev), tri.to(dev)
    out = {}
    for prec in ("fp32", "3xtf32", "tf32+bf16x2", "tf32"):
        got = engine.score_1vsN(model, "sp_", e, r, e, t[:, 0].contiguous(), t[:, 1].contiguous(), None, 1.0, prec)
        out[prec] = float((got.cpu().double() - ref).abs().max()) / rms
    print(json.dumps({"case": "parity vs fp64 (max|d|/rms)", **out}), flush=True)


CASES = {
    "parity": case_parity,
    "tc3_step": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "3xtf32", "step"),
    "tc3_store": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "3xtf32", "store"),
    "tc3_kl": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "3xtf32", "kl"),
    "tc3_store_n512": lambda: case_1vsall("complex", 14541, 237, 512, 512, "3xtf32", "store"),
    "mix_step": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "tf32+bf16x2", "step"),
    "mix_store": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "tf32+bf16x2", "store"),
    "mix_kl": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "tf32+bf16x2", "kl"),
    "mix_step_n4096": lambda: case_1vsall("complex", 14541, 237, 512, 4096, "tf32+bf16x2", "step"),
    "mix_rescal": lambda: case_1vsall("rescal", 123182, 37, 200, 1024, "tf32+bf16x2", "step"),
    "tc1_step": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "tf32", "step"),
    "tc1_store": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "tf32", "store"),
    "fp32_step": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "fp32", "step"),
    "fp32_store": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "fp32", "store"),
    "tc3_step_n128": lambda: case_1vsall("complex", 14541, 237, 512, 128, "3xtf32", "step"),
    "tc3_step_n4096": lambda: case_1vsall("complex", 14541, 237, 512, 4096, "3xtf32", "step"),
    "rescal_step": lambda: case_1vsall("rescal", 123182, 37, 200, 1024, "3xtf32", "step"),
    # the default pre-split fp16 path ("auto") at the shapes of the explicit-precision cases above
    "auto_step": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "auto", "step"),
    "auto_store": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "auto", "store"),
    "auto_kl": lambda: case_1vsall("complex", 14541, 237, 512, 1024, "auto", "kl"),
    "auto_step_n128": lambda: case_1vsall("complex", 14541, 237, 512, 128, "auto", "step"),
    "auto_step_n4096": lambda: case_1vsall("complex", 14541, 237, 512, 4096, "auto", "step"),
    "auto_store_n128": lambda: case_1vsall("complex", 14541, 237, 512, 128, "auto", "store"),
    "auto_store_n4096": lambda: case_1vsall("complex", 14541, 237, 512, 4096, "auto", "store"),
    "auto_kl_n128": lambda: case_1vsall("complex", 14541, 237, 512, 128, "auto", "kl"),
    "auto_kl_n4096": lambda: case_1vsall("complex", 14541, 237, 512, 4096, "auto", "kl"),
    "auto_rescal_step": lambda: case_1vsall("rescal", 123182, 37, 200, 1024, "auto", "step"),
    "transe_step": lambda: case_1vsall("transe", 14541, 237, 512, 1024, "auto", "step"),
    "transe_store": lambda: case_1vsall("transe", 14541, 237, 512, 1024, "auto", "store"),
    "rotate_step": lambda: case_1vsall("rotate", 14541, 237, 512, 1024, "auto", "step"),
    "transe_wiki_shard": lambda: case_1vsall("transe", 600000, 822, 512, 128, "auto", "store"),
    "kvsall_rescal": lambda: case_kvsall("rescal", 123182, 37, 200, 512, "bce"),
    "kvsall_rescal_kl": lambda: case_kvsall("rescal", 123182, 37, 200, 512, "kl"),
    "ns_rotate": lambda: case_ns("rotate", 40943, 11, 512, 512, 1000),
    "ns_complex": lambda: case_ns("complex", 40943, 11, 512, 512, 1000),
}

if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    for nm in names:
        try:
            CASES[nm]()
        except Exception as e:  # keep going: this is a survey
            print(json.dumps({"case": nm, "error": repr(e)[:300]}), flush=True)
