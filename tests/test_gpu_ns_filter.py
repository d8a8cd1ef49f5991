"""Filtered negative sampling on the H100: b200kge_sample_uniform_filtered bit for bit against the numpy mirror
(tests/ns_filter_oracle.py), its distribution, and B200TrainingJobNegativeSampling with `negative_sampling.filtering.*`
and `user.b200_device_sampling` against the unmodified reference job fed the same negatives."""
import numpy as np
import pytest
import torch

import ns_filter_oracle as nfo
from kge_b200 import hostenv
from kge_b200.indexing import index_KvsAll

pytestmark = pytest.mark.gpu
S, P, O = 0, 1, 2
PAIR = {S: "po", P: "so", O: "sp"}


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    assert torch.cuda.is_available() and engine.device_ok()
    return engine


def _zipf_split(E, R, N, seed):
    """Triples with Zipf-distributed entities and relations (heavy keys), plus repeats of the first 100."""
    g = np.random.default_rng(seed)
    s = (g.zipf(1.3, N) - 1) % E
    o = (g.zipf(1.3, N) - 1) % E
    p = (g.zipf(1.5, N) - 1) % R
    t = torch.from_numpy(np.stack([s, p, o], 1).astype(np.int64))
    return torch.cat([t, t[:100]])


def _index(eng, split, slot, vocab):
    return eng.FilterIndex(index_KvsAll(split, PAIR[slot]), vocab, "cuda")


def _check(eng, n, K, vocab, seed, offset, tri, slot, index):
    got = eng.sample_uniform_filtered(n, K, vocab, seed, offset, tri.cuda(), slot, index).cpu().numpy()
    want, replaced = nfo.sample_uniform_filtered(n, K, vocab, seed, offset, tri.numpy(), slot, index.keys.cpu().numpy(),
                                                 index.offsets.cpu().numpy(), index.values.cpu().numpy(),
                                                 return_replaced=True)
    assert np.array_equal(got, want)
    # every position the filter left alone is sample_uniform's draw
    plain = eng.sample_uniform(n, K, vocab, seed, offset, "cuda").cpu().numpy()
    assert np.array_equal(got[~replaced], plain[~replaced])
    return got, replaced


@pytest.mark.parametrize("slot", [S, P, O])
@pytest.mark.parametrize("n,K", [(3, 7), (512, 1000)])
def test_entry_matches_the_mirror(eng, slot, n, K):
    E, R = 40943, 11
    split = _zipf_split(E, R, 86835, 1 + slot)
    vocab = R if slot == P else E
    index = _index(eng, split, slot, vocab)         # P slot: some (s, o) keys hold all 11 relations (rows of -1)
    tri = split[torch.randperm(len(split), generator=torch.Generator().manual_seed(slot))[:n]]
    for seed, offset in ((7, 0), (2 ** 40 + 1, (3 << 2) | slot)):
        got, replaced = _check(eng, n, K, vocab, seed, offset, tri, slot, index)
        if n == 512:
            assert replaced.any()
            # no output is a positive of its row's key: exhaustive against the host index
            pos = nfo.positives_of(split, slot)
            a, b = nfo.KEY_COLS[slot]
            for i in range(n):
                p = pos.get((int(tri[i, a]), int(tri[i, b])))
                if p:
                    assert not np.isin(got[i], np.fromiter(p, np.int64)).any()


def test_entry_at_a_large_vocabulary(eng):
    """V = 4.8M with a key holding half of the vocabulary."""
    V = 4_800_000
    g = torch.Generator().manual_seed(3)
    heavy = torch.randperm(V, generator=g)[: V // 2]
    split = torch.cat([torch.stack([torch.zeros_like(heavy), torch.zeros_like(heavy), heavy], 1),
                       torch.stack([torch.randint(0, V, (50000,), generator=g), torch.randint(0, 5, (50000,), generator=g),
                                    torch.randint(0, V, (50000,), generator=g)], 1)])
    index = _index(eng, split, O, V)
    tri = torch.cat([torch.zeros((256, 3), dtype=torch.int64), split[-256:]])
    got, replaced = _check(eng, 512, 1000, V, 11, 5, tri, O, index)
    assert replaced[:256].mean() > 0.4
    assert not np.isin(got[:256], heavy.numpy()).any()


def test_absent_empty_and_saturated_keys(eng):
    """An absent key and a key listed without values are unfiltered; m = V - 1 gives the one remaining id everywhere;
    m = V gives -1."""
    V, K = 40, 300
    index = eng.FilterIndex(index_KvsAll(torch.zeros((0, 3), dtype=torch.int64), "sp"), V, "cuda")
    # keys (0,0): m = V - 1 (all but 17), (0,1): no values, (0,2): m = V, (0,3): {5}
    vals = [v for v in range(V) if v != 17] + list(range(V)) + [5]
    index.keys = torch.tensor([[0, 0], [0, 1], [0, 2], [0, 3]], device="cuda")
    index.offsets = torch.tensor([0, V - 1, V - 1, 2 * V - 1, 2 * V], device="cuda")
    index.values = torch.tensor(vals, device="cuda")
    tri = torch.tensor([[0, 0, 9], [0, 1, 9], [0, 2, 9], [0, 3, 9], [1, 0, 9]])
    got = eng.sample_uniform_filtered(5, K, V, 4, 2, tri.cuda(), O, index).cpu().numpy()
    want = nfo.sample_uniform_filtered(5, K, V, 4, 2, tri.numpy(), O, index.keys.cpu().numpy(),
                                       index.offsets.cpu().numpy(), index.values.cpu().numpy())
    assert np.array_equal(got, want)
    plain = eng.sample_uniform(5, K, V, 4, 2, "cuda").cpu().numpy()
    assert (got[0] == 17).all()
    assert np.array_equal(got[1], plain[1]) and np.array_equal(got[4], plain[4])
    assert (got[2] == -1).all()
    assert 5 not in got[3] and np.array_equal(got[3][plain[3] != 5], plain[3][plain[3] != 5])


def test_distribution_over_the_non_positives(eng):
    """V = 50, m = 30, 10^6 draws, fixed seed: chi-square over the 20 non-positives."""
    from scipy.stats import chisquare

    V, m = 50, 30
    pos = torch.from_numpy(np.sort(np.random.default_rng(0).choice(V, m, replace=False)))
    split = torch.stack([torch.zeros_like(pos), torch.zeros_like(pos), pos], 1)
    index = _index(eng, split, O, V)
    got = eng.sample_uniform_filtered(1000, 1000, V, 123, 9, torch.zeros((1000, 3), dtype=torch.int64).cuda(), O,
                                      index).cpu().numpy()
    assert not np.isin(got, pos.numpy()).any()
    counts = np.bincount(got.reshape(-1), minlength=V)[np.setdiff1d(np.arange(V), pos.numpy())]
    assert chisquare(counts).pvalue > 1e-3


# ---- the job against the reference job ---------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 211, 5, 32
TOL = 1e-4
P_ENT, P_REL = 0.3, 0.1


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    sp = ju.synthetic_splits(JE, JR, 600, 60, 60)
    k = torch.arange(40, dtype=sp["train"].dtype)              # heavy keys: (0, 0, ?) and (?, 1, 1)
    sp["train"] = torch.cat([sp["train"], torch.stack([0 * k, 0 * k, k], 1), torch.stack([k, 0 * k + 1, 0 * k + 1], 1),
                             sp["train"][:20]])
    return sp


def _close(got, ref, what, tol):
    got, ref = got.double(), ref.double()
    rms = max(float(ref.pow(2).mean().sqrt()), 1e-6)
    err = float((got - ref).abs().max())
    assert err <= tol * rms, f"{what}: max|d|={err:.3e} rms={rms:.3e}"


def _train_pair(splits, filt, recip=False, dropout=False, monkeypatch=None):
    import jobs_util as ju
    from kge_b200 import engine

    import ns_dropout_oracle as nso

    cfg = {"negative_sampling.implementation": "triple", "negative_sampling.num_samples.s": 7,
           "negative_sampling.num_samples.o": 9, "train.optimizer.default.type": "SGD",
           "train.optimizer.default.args.lr": 0.1}
    cfg.update({f"negative_sampling.filtering.{c}": True for c in filt})
    drawn, filtered = {S: [], O: []}, []
    for name in ("sample_uniform", "sample_uniform_filtered"):
        orig = getattr(engine, name)

        def spy(*a, orig=orig, name=name, **kw):
            out = orig(*a, **kw)
            slot = a[-2] if name == "sample_uniform_filtered" else (a[4] & 3)
            drawn[slot].append(out.cpu())
            if name == "sample_uniform_filtered":
                filtered.append((slot, a[5].cpu(), out.cpu()))
            return out
        monkeypatch.setattr(engine, name, spy)

    def make(tag, dev):
        m = "complex" if tag == "ref" else "b200_complex"
        c = dict(cfg)
        imports = ()
        model = m
        if recip:
            c["reciprocal_relations_model.base_model.type"] = m
            model, imports = "reciprocal_relations_model", (m,)
        if dropout:
            c.update({f"{m}.entity_embedder.dropout": P_ENT, f"{m}.relation_embedder.dropout": P_REL})
        if tag == "b200":
            c["user.b200_device_sampling"] = True
            if dropout:
                c["user.b200_ns_dropout"] = True
        return ju.make_job(model, JE, JR, JD, splits, device=dev, train_type="negative_sampling", loss="kl",
                           batch_size=64, forward_only=False, extra=c, imports=imports,
                           job_class="B200TrainingJobNegativeSampling" if tag == "b200" else None)

    torch.manual_seed(0)
    init = make("ref", "cpu")
    out = {}
    for tag, dev in (("b200", "cuda"), ("ref", "cuda")):
        job = make(tag, dev)
        with torch.no_grad():
            for a, b in zip(init.model.parameters(), job.model.parameters()):
                b.copy_(a.to(b.device))
        if tag == "b200":
            assert job._device_sampling and sorted(job._filter_index) == sorted("spo".index(c) for c in filt)
        else:
            if dropout:
                nso.patch_reference_ns_job(job, P_ENT, P_REL)
            queue = {slot: list(v) for slot, v in drawn.items()}
            # the reference draws the same negatives; its own filter then finds no positive to replace
            job._sampler._sample = lambda tri, slot, num: (queue[slot].pop(0)[: len(tri), :num].clone() if num > 0
                                                           else torch.empty((len(tri), 0), dtype=torch.int64))
        losses = []
        for ep in range(2):
            job.epoch += 1
            if job.loader is None:
                job._prepare()
            ju.seed_all(10 + ep)
            losses.append(job.run_epoch()["avg_loss"])
        if tag == "ref":
            assert not any(queue.values())                        # every device-drawn batch was consumed
        out[tag] = (losses, [p.detach().cpu() for p in job.model.parameters()])
    return out, filtered


@needs_ref
@pytest.mark.parametrize("filt,recip,dropout", [("o", False, False), ("so", False, False), ("so", True, False),
                                                ("so", False, True)])
def test_job_matches_the_reference_job(eng, splits, filt, recip, dropout, monkeypatch):
    out, filtered = _train_pair(splits, filt, recip, dropout, monkeypatch)
    assert out["b200"][0][0] == pytest.approx(out["ref"][0][0], rel=TOL)
    assert out["b200"][0][1] == pytest.approx(out["ref"][0][1], rel=1e-3)
    for k, (a, b) in enumerate(zip(out["b200"][1], out["ref"][1])):
        _close(a, b, f"parameter {k}", 10 * TOL)
    # no negative drawn in the epochs is a positive of the filtering split; the keys are the dataset's triples, also
    # under the reciprocal wrapper
    assert sorted({c[0] for c in filtered}) == sorted("spo".index(c) for c in filt)
    pos = {slot: nfo.positives_of(splits["train"], slot) for slot in (S, O)}
    for slot, tri, neg in filtered:
        a, b = nfo.KEY_COLS[slot]
        assert (neg >= 0).all() and (neg < JE).all()
        for i in range(len(tri)):
            p = pos[slot].get((int(tri[i, a]), int(tri[i, b])), set())
            assert not set(neg[i].tolist()) & p
