"""Frequency negative sampling on the H100: b200kge_sample_frequency and b200kge_sample_frequency_filtered bit for bit
against the numpy mirror (tests/ns_frequency_oracle.py), against the uniform entries under equal weights, their
distributions, and B200TrainingJobNegativeSampling with `negative_sampling.sampling_type: frequency` and
`user.b200_device_sampling` against the unmodified reference job fed the same negatives."""
import numpy as np
import pytest
import torch

import ns_filter_oracle as nfo
import ns_frequency_oracle as nfq
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


_SPLITS = {}


def _zipf_split(E, R, N, seed):
    """Triples with Zipf-distributed entities and relations (heavy keys and heavy ids), plus repeats of the first 100."""
    if (E, R, N, seed) not in _SPLITS:
        g = np.random.default_rng(seed)
        s = (g.zipf(1.3, N) - 1) % E
        o = (g.zipf(1.3, N) - 1) % E
        p = (g.zipf(1.5, N) - 1) % R
        t = torch.from_numpy(np.stack([s, p, o], 1).astype(np.int64))
        _SPLITS[(E, R, N, seed)] = torch.cat([t, t[:100]])
    return _SPLITS[(E, R, N, seed)]


def _tables(eng, split, slot, vocab, alpha):
    table = eng.FrequencyTable(torch.bincount(split[:, slot], minlength=vocab), alpha, "cuda")
    index = table.attach(eng.FilterIndex(index_KvsAll(split, PAIR[slot]), vocab, "cuda"))
    return table, index


def _check(eng, n, K, table, seed, offset, tri, slot, index):
    """Both entries against the mirror; the filtered entry's unreplaced positions against the unfiltered entry."""
    cdf = table.cdf.cpu().numpy()
    plain = eng.sample_frequency(n, K, table, seed, offset).cpu().numpy()
    assert np.array_equal(plain, nfq.sample_frequency(n, K, cdf, seed, offset))
    got = eng.sample_frequency_filtered(n, K, table, seed, offset, tri.cuda(), slot, index).cpu().numpy()
    want, replaced = nfq.sample_frequency_filtered(
        n, K, cdf, seed, offset, tri.numpy(), slot, index.keys.cpu().numpy(), index.offsets.cpu().numpy(),
        index.values.cpu().numpy(), index.below.cpu().numpy(), return_replaced=True)
    assert np.array_equal(got, want)
    assert np.array_equal(got[~replaced], plain[~replaced])
    return plain, got, replaced


SHAPES = {"wn18rr": (40943, 11, 86835), "wikidata5m": (4_800_000, 822, 2_000_000)}


@pytest.mark.parametrize("shape", ["wn18rr", "wikidata5m"])
@pytest.mark.parametrize("alpha", [0, 1, 0.5])
@pytest.mark.parametrize("n,K", [(3, 7), (512, 1000)])
@pytest.mark.parametrize("slot", [S, P, O])
def test_entries_match_the_mirror(eng, shape, alpha, n, K, slot):
    E, R, N = SHAPES[shape]
    split = _zipf_split(E, R, N, 1)
    vocab = R if slot == P else E
    table, index = _tables(eng, split, slot, vocab, alpha)
    if alpha == 0 and slot != P:
        assert (torch.diff(table.cdf.cpu()) == 0).any()          # entities of zero weight exist
    tri = split[torch.randperm(len(split), generator=torch.Generator().manual_seed(slot))[:n]]
    for seed, offset in ((7, 0), (2 ** 40 + 1, (3 << 2) | slot)):
        plain, got, replaced = _check(eng, n, K, table, seed, offset, tri, slot, index)
        q = torch.diff(table.cdf.cpu()).numpy()
        assert (q[plain] > 0).all() and (q[got[got >= 0]] > 0).all()       # never an id of zero weight
        if n == 512:
            assert replaced.any()
        if n == 512 and shape == "wn18rr":
            # no output is a positive of its row's key: exhaustive against the split
            pos = nfo.positives_of(split, slot)
            a, b = nfo.KEY_COLS[slot]
            for i in range(n):
                p = pos.get((int(tri[i, a]), int(tri[i, b])))
                if p and (got[i] >= 0).all():
                    assert not np.isin(got[i], np.fromiter(p, np.int64)).any()


def test_rows_whose_positives_carry_all_the_weight(eng):
    """smoothing 0: ids 0..9 only have weight; key (0, 0) holds all of them (-1), key (0, 1) all but id 4."""
    V, K = 1000, 300
    tri = [[i, 2, i] for i in range(10)] + [[0, 0, i] for i in range(10)] + [[0, 1, i] for i in range(10) if i != 4]
    split = torch.tensor(tri)
    table, index = _tables(eng, split, O, V, 0)
    assert index.full_keys == 1 and index.first_full_key == (0, 0)
    rows = torch.tensor([[0, 0, 9], [0, 1, 9], [5, 2, 9], [7, 3, 9]])
    plain, got, _ = _check(eng, 4, K, table, 4, 2, rows, O, index)
    assert (got[0] == -1).all() and (got[1] == 4).all()
    assert np.array_equal(got[3], plain[3]) and not np.isin(got[2], [5]).any()


@pytest.mark.parametrize("V", [11, 40943, 4_800_000])
def test_equal_weights_reproduce_the_uniform_entries(eng, V):
    split = _zipf_split(40943, 11, 86835, 2)
    split = split % torch.tensor([V, 11, V])
    for counts, alpha in ((torch.zeros(V, dtype=torch.int64), 1), (torch.full((V,), 3), 0)):
        table = eng.FrequencyTable(counts, alpha, "cuda")
        index = table.attach(eng.FilterIndex(index_KvsAll(split, PAIR[O]), V, "cuda"))
        tri = split[:512].cuda()
        for seed, offset in ((3, 1), (2 ** 50 + 1, 77)):
            assert torch.equal(eng.sample_frequency(512, 1000, table, seed, offset),
                               eng.sample_uniform(512, 1000, V, seed, offset, "cuda"))
            assert torch.equal(eng.sample_frequency_filtered(512, 1000, table, seed, offset, tri, O, index),
                               eng.sample_uniform_filtered(512, 1000, V, seed, offset, tri, O, index))


def test_distributions(eng):
    """10^6 draws, fixed seed: chi-square of the unfiltered draws against q / Q, and of a heavy key's filtered draws
    against the complement law q_y / (Q - M)."""
    from scipy.stats import chisquare

    V = 50
    counts = torch.from_numpy(np.random.default_rng(2).integers(0, 40, V))
    heavy = torch.from_numpy(np.sort(np.argsort(-counts.numpy())[:20]))  # the 20 heaviest ids, positives of (0, 0)
    split = torch.stack([torch.zeros_like(heavy), torch.zeros_like(heavy), heavy], 1)
    table = eng.FrequencyTable(counts, 1, "cuda")
    index = table.attach(eng.FilterIndex(index_KvsAll(split, PAIR[O]), V, "cuda"))
    q = torch.diff(table.cdf.cpu()).double().numpy()
    got = eng.sample_frequency(1000, 1000, table, 123, 9).cpu().numpy()
    assert chisquare(np.bincount(got.reshape(-1), minlength=V), q / q.sum() * got.size).pvalue > 1e-3
    got = eng.sample_frequency_filtered(1000, 1000, table, 123, 9, torch.zeros((1000, 3), dtype=torch.int64).cuda(),
                                        O, index).cpu().numpy()
    assert not np.isin(got, heavy.numpy()).any()
    rest = np.setdiff1d(np.arange(V), heavy.numpy())
    obs = np.bincount(got.reshape(-1), minlength=V)[rest]
    assert chisquare(obs, q[rest] / q[rest].sum() * got.size).pvalue > 1e-3


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
    """Two epochs of the b200 job with frequency sampling on the device, and of the reference job (uniform sampler)
    whose `_sample` replays the device's draws."""
    import jobs_util as ju
    from kge_b200 import engine

    import ns_dropout_oracle as nso

    cfg = {"negative_sampling.implementation": "triple", "negative_sampling.num_samples.s": 7,
           "negative_sampling.num_samples.o": 9, "train.optimizer.default.type": "SGD",
           "train.optimizer.default.args.lr": 0.1}
    cfg.update({f"negative_sampling.filtering.{c}": True for c in filt})
    drawn, filtered = {S: [], O: []}, []
    for name in ("sample_frequency", "sample_frequency_filtered"):
        orig = getattr(engine, name)

        def spy(*a, orig=orig, name=name, **kw):
            out = orig(*a, **kw)
            slot = a[6] if name == "sample_frequency_filtered" else (a[4] & 3)
            drawn[slot].append(out.cpu())
            if name == "sample_frequency_filtered":
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
            c["negative_sampling.sampling_type"] = "frequency"
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
            assert job._device_sampling and sorted(job._frequency) == [S, O]
            assert sorted(job._filter_index) == sorted("spo".index(c) for c in filt)
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
    return out, filtered, drawn


@needs_ref
@pytest.mark.parametrize("filt,recip,dropout", [("", False, False), ("o", False, False), ("so", False, False),
                                                ("so", True, False), ("o", False, True)])
def test_job_matches_the_reference_job(eng, splits, filt, recip, dropout, monkeypatch):
    out, filtered, drawn = _train_pair(splits, filt, recip, dropout, monkeypatch)
    assert out["b200"][0][0] == pytest.approx(out["ref"][0][0], rel=TOL)
    assert out["b200"][0][1] == pytest.approx(out["ref"][0][1], rel=1e-3)
    for k, (a, b) in enumerate(zip(out["b200"][1], out["ref"][1])):
        _close(a, b, f"parameter {k}", 10 * TOL)
    assert sorted({c[0] for c in filtered}) == sorted("spo".index(c) for c in filt)
    # the draws follow the training split's frequencies: the heavy object 1 of the (?, 1, 1) block is drawn far more
    # often than uniform sampling would (1 / 211)
    o = torch.cat([d.reshape(-1) for d in drawn[O]])
    assert (o >= 0).all() and (o < JE).all() and float((o == 1).double().mean()) > 5 / JE
    pos = {slot: nfo.positives_of(splits["train"], slot) for slot in (S, O)}
    for slot, tri, neg in filtered:
        a, b = nfo.KEY_COLS[slot]
        for i in range(len(tri)):
            p = pos[slot].get((int(tri[i, a]), int(tri[i, b])), set())
            assert not set(neg[i].tolist()) & p
