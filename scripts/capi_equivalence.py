"""Runs every host path of the C entry points on seeded inputs against one built source tree, and compares such runs.

    python scripts/capi_equivalence.py run TREE OUT.npz
    python scripts/capi_equivalence.py compare BASE_1.npz BASE_2.npz [BASE_3.npz ...] NEW.npz [--json OUT.json]

`run` imports kge_b200 from TREE and saves, per call, every output and the number of kernel launches the call issued
(b200kge_launch_count).  `compare` takes two or more runs of a baseline tree and one of a changed tree: an output every
baseline run reproduces bit for bit must be bit-identical in the changed tree, any other output must lie within the
baseline's own run-to-run spread (largest max |difference| between two of its runs), and every launch count must be
equal.  Gradients scattered with atomics vary from run to run, so give enough baseline runs to bound that spread.  Paths: the 1vsAll training step forward
and backward of every model for BCE and KL, plain, under dropout, with reciprocal relations and both; the backward of a
dense score block; the KvsAll CSR loss and its backward with and without dropout (on the _po streams too), for the dot
family and for TransE L1 / L2 and RotatE L1; the evaluation ranking; the default-precision scorers; negative sampling:
the scores of the S and O slots, plain and with dropout (`triple`, `batch`), and their backward in BCE, given-gradient
and dropout form for ComplEx, TransE L1 / L2 and RotatE L1.
"""
import argparse
import json
import sys

import numpy as np

MODELS = ("complex", "distmult", "simple", "cp", "rescal", "transe", "rotate")
E, R, D, N = 2000, 11, 64, 256


def run(tree, out):
    sys.path.insert(0, tree)
    import torch
    from kge_b200 import engine as eng

    assert eng.device_ok()
    g = torch.Generator().manual_seed(20261016)
    dev = "cuda"

    def tables(model, rel_rows):
        rd = D * D if model == "rescal" else D
        ent = (torch.randn(E, D, generator=g) * 0.3).to(dev)
        rel = (torch.randn(rel_rows, rd, generator=g) * (0.3 / D if model == "rescal" else 0.3)).to(dev)
        return ent, rel

    tri = torch.stack([torch.randint(0, E, (N,), generator=g), torch.randint(0, R, (N,), generator=g),
                       torch.randint(0, E, (N,), generator=g)], 1).to(dev)
    s, p, o = (tri[:, i].contiguous() for i in range(3))
    key = eng.DropoutKey(0.2, 0.1, 7, 3)
    res = {}

    def rec(name, fn):
        torch.cuda.synchronize()
        eng.launch_count(reset=True)
        try:
            got = fn()
        except Exception as e:      # a refused call is an outcome to compare too
            got = torch.tensor(list(f"{type(e).__name__}: {e}".encode()), dtype=torch.uint8)
        torch.cuda.synchronize()
        res["launches/" + name] = np.array([eng.launch_count()])
        got = got if isinstance(got, tuple) else (got,)
        for i, t in enumerate(got):
            res[f"{name}/{i}"] = t.detach().cpu().numpy()

    for model in MODELS:
        ent, rel = tables(model, R)
        ent2, rel2 = tables(model, 2 * R)
        for loss in ("bce", "kl"):
            for mode in ("plain", "dropout", "reciprocal", "reciprocal+dropout"):
                drop = key if "dropout" in mode else None
                nm = f"train/{model}/{loss}/{mode}"
                if mode.startswith("reciprocal"):
                    rec(nm + "/fwd", lambda: eng.train_1vsall_reciprocal_forward(model, ent2, rel2, tri, R, loss,
                                                                                 dropout=drop))
                    rec(nm + "/bwd", lambda: eng.train_1vsall_reciprocal_backward(model, ent2, rel2, tri, R, loss,
                                                                                  dropout=drop))
                else:
                    rec(nm + "/fwd", lambda: eng.train_1vsall_forward(model, ent, rel, tri, loss, dropout=drop))
                    rec(nm + "/bwd", lambda: eng.train_1vsall_backward(model, ent, rel, tri, loss, dropout=drop))
        # default-precision scorers
        sub = torch.randperm(E, generator=g)[:700].to(dev)
        rec(f"score/{model}/sp_po", lambda: eng.score_sp_po(model, ent, rel, s, p, o))
        rec(f"score/{model}/po_subset", lambda: eng.score_1vsN(model, "_po", ent, rel, ent, o, p, sub))
        rec(f"score/{model}/sp_loss", lambda: eng.score_1vsN_loss(model, "sp_", ent, rel, ent, o, s, p, loss="kl"))
        # the evaluation ranking, plain and reciprocal
        for nr, (et, rt) in ((0, (ent, rel)), (R, (ent2, rel2))):
            true = torch.randn(2 * N, generator=g).to(dev)
            own = torch.cat([o, s])
            offs = torch.arange(0, 2 * N + 1, dtype=torch.int64, device=dev)
            rec(f"rank_eval/{model}/num_rel{nr}",
                lambda: eng.rank_sp_po_eval(model, et, rt, s, p, o, true, own, offs, own, num_relations=nr))
    # backward of a dense score block
    for model, l_norm in (("distmult", 1.0), ("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)):
        ent, rel = tables(model, R)
        gs = torch.randn(N, E, generator=g).to(dev)
        for comb, q in (("sp_", s), ("_po", o)):
            rec(f"score_bwd/{model}/l{l_norm:g}/{comb}",
                lambda: eng.score_1vsN_backward(model, comb, ent, rel, q, p, gs, l_norm=l_norm))
    # KvsAll CSR losses
    cnt = torch.randint(1, 4, (N,), generator=g)
    offs = torch.cat([torch.zeros(1, dtype=torch.int64), cnt.cumsum(0)]).to(dev)
    cols = torch.cat([torch.randperm(E, generator=g)[:int(c)].sort().values for c in cnt]).to(dev)
    for model in ("complex", "distmult", "rescal"):
        ent, rel = tables(model, 2 * R)
        for loss in ("kl", "bce"):
            for ls in (0.0, 0.1):
                for drop, streams in ((None, None), (key, None), (key, "_po")):
                    nm = f"csr/{model}/{loss}/ls{ls}/{'drop' if drop else 'plain'}{streams or ''}"
                    rec(nm + "/fwd", lambda: eng.score_1vsN_loss_csr(model, "sp_", ent, rel, ent, offs, cols, q=s, p=p,
                                                                     loss=loss, label_smoothing=ls, dropout=drop,
                                                                     dropout_streams=streams, return_rows=True))
                    rec(nm + "/bwd", lambda: eng.score_1vsN_loss_csr_backward(model, "sp_", ent, rel, s, p, offs, cols,
                                                                              loss=loss, label_smoothing=ls,
                                                                              dropout=drop, dropout_streams=streams))
    # the KvsAll CSR loss and its backward for the distance family
    for model, l_norm in (("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)):
        ent, rel = tables(model, 2 * R)
        for loss in ("kl", "bce"):
            for ls in (0.0, 0.1):
                for drop, streams in ((None, None), (key, None), (key, "_po")):
                    nm = f"csr/{model}/l{l_norm:g}/{loss}/ls{ls}/{'drop' if drop else 'plain'}{streams or ''}"
                    rec(nm + "/fwd", lambda: eng.score_1vsN_loss_csr(model, "sp_", ent, rel, ent, offs, cols, q=s, p=p,
                                                                     loss=loss, label_smoothing=ls, l_norm=l_norm,
                                                                     dropout=drop, dropout_streams=streams,
                                                                     return_rows=True))
                    rec(nm + "/bwd", lambda: eng.score_1vsN_loss_csr_backward(model, "sp_", ent, rel, s, p, offs, cols,
                                                                              loss=loss, label_smoothing=ls,
                                                                              dropout=drop, dropout_streams=streams,
                                                                              l_norm=l_norm))
    # negative sampling: the scores of a slot and its backward (BCE in the kernel, a given gradient, dropout)
    K = 16
    negs = torch.randint(0, E, (N, K), generator=g).to(dev)
    grads = {slot: (torch.randn(N, K + 1, generator=g) * 0.01).to(dev) for slot in (0, 2)}
    for model, l_norm in (("complex", 1.0), ("transe", 1.0), ("transe", 2.0), ("rotate", 1.0)):
        ent, rel = tables(model, R)
        for slot in (0, 2):
            nm = f"ns/{model}/l{l_norm:g}/slot{slot}"
            rec(nm + "/score", lambda: eng.ns_score(model, ent, rel, tri, negs, slot, with_positive=True, l_norm=l_norm))
            rec(nm + "/bwd_bce", lambda: eng.ns_backward(model, ent, rel, tri, {slot: negs}, offset=0.5, l_norm=l_norm))
            rec(nm + "/bwd_grad", lambda: eng.ns_backward(model, ent, rel, tri, {slot: negs}, l_norm=l_norm,
                                                          grad_scores=grads))
            for impl in ("triple", "batch"):
                rec(nm + f"/score_drop_{impl}", lambda: eng.ns_score(model, ent, rel, tri, negs, slot, with_positive=True,
                                                                     l_norm=l_norm, dropout=key, implementation=impl))
                rec(nm + f"/bwd_drop_{impl}", lambda: eng.ns_backward(model, ent, rel, tri, {slot: negs}, l_norm=l_norm,
                                                                      grad_scores=grads, dropout=key,
                                                                      implementation=impl))
    np.savez(out, **res)
    print(f"{len(res)} arrays -> {out}")


def compare(base_paths, c_path, json_out=None):
    bases, c = [np.load(p) for p in base_paths], np.load(c_path)
    keys = sorted(bases[0].files)
    assert all(set(keys) == set(x.files) for x in bases + [c]), set(keys) ^ set(c.files)
    bad, spread_keys = [], []

    def same(x, y):
        return x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes()

    def maxdiff(x, y):
        return float(np.max(np.abs(x.astype(np.float64) - y.astype(np.float64)))) if x.size else 0.0

    for k in keys:
        xs, z = [x[k] for x in bases], c[k]
        if k.startswith("launches/"):
            if len({int(v[0]) for v in xs + [z]}) != 1:
                bad.append((k, "launch count", [int(v[0]) for v in xs + [z]]))
        elif all(same(xs[0], x) for x in xs[1:]):
            if not same(xs[0], z):
                bad.append((k, "baseline reproducible but new differs", maxdiff(xs[0], z)))
        else:
            spread = max(maxdiff(x, y) for i, x in enumerate(xs) for y in xs[i + 1:])
            d = min(maxdiff(z, x) for x in xs)
            spread_keys.append((k, spread, d))
            if z.shape != xs[0].shape or d > spread:
                bad.append((k, "outside the baseline's spread", d, spread))
    summary = {"arrays": len(keys), "bit_identical_in_baseline": len(keys) - len(spread_keys),
               "nondeterministic_in_baseline": spread_keys, "failures": bad, "ok": not bad}
    text = json.dumps(summary, indent=1)
    print(text)
    if json_out:
        with open(json_out, "w") as fh:
            fh.write(text + "\n")
    return 0 if not bad else 1


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("tree")
    r.add_argument("out")
    c = sub.add_parser("compare")
    c.add_argument("bases", nargs="+", help="two or more runs of the baseline tree")
    c.add_argument("new")
    c.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.cmd == "run":
        run(args.tree, args.out)
        return 0
    assert len(args.bases) >= 2, "the baseline's spread needs at least two of its runs"
    return compare(args.bases, args.new, args.json)


if __name__ == "__main__":
    sys.exit(main())
