"""Frequency negative sampling on the CPU: the host builders of the integer weights and of the filtered entry's
per-entry table (through ctypes), the numpy mirror of b200kge_sample_frequency(_filtered)
(tests/ns_frequency_oracle.py) checked exhaustively at tiny total weight and against a plain-Python restatement, and
B200TrainingJobNegativeSampling's routing of `negative_sampling.sampling_type: frequency` with
`user.b200_device_sampling`.  The kernels are checked against the same mirror in tests/test_gpu_ns_frequency.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import ns_filter_oracle as nfo
import ns_frequency_oracle as nfq
from kge_b200 import engine, hostenv
from kge_b200.indexing import filter_csr, frequency_below, frequency_cdf, index_KvsAll

S, P, O = 0, 1, 2
PAIR = {S: "po", P: "so", O: "sp"}
INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from kge_b200 import _lib
    from kge_b200.build import build_native

    build_native()
    return _lib.load()


def _zipf_counts(V, N, seed):
    g = np.random.default_rng(seed)
    return torch.from_numpy(np.bincount((g.zipf(1.2, N) - 1) % V, minlength=V).astype(np.int64))


# ---- the weights --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.5, 3.0, 1e-3, 2.0 ** -40])
@pytest.mark.parametrize("V,N", [(7, 30), (1000, 20000), (40943, 86835)])
def test_cdf_is_the_prefix_of_the_quantised_weights(alpha, V, N):
    counts = _zipf_counts(V, N, V)
    cdf = frequency_cdf(counts, alpha).numpy()
    q, s = nfq.quantise(counts.tolist(), alpha)
    assert cdf[0] == 0 and cdf.dtype == np.int64
    assert np.diff(cdf).tolist() == q
    Q = int(cdf[-1])
    assert 0 < Q <= 2 ** 62
    assert sum(nfq._quantised(counts.tolist(), alpha, s + 1)) > 2 ** 62        # s is the largest scale that fits
    if alpha == int(alpha):
        # exactly proportional to the reference's weights counts + alpha
        assert q == [(int(c) + int(alpha)) << s for c in counts]
    else:
        w = counts.double().numpy() + alpha
        rel = np.abs(np.array(q, dtype=np.float64) / 2.0 ** s - w) / w
        assert rel.max() <= 2.0 ** -s / w.min()
    if alpha == 0:
        assert all((qq == 0) == (int(c) == 0) for qq, c in zip(q, counts))


def test_cdf_at_a_wikidata5m_scale():
    """V = 4.8M ids, 20.6M training triples: relative error per id of the fractional smoothing near 2^-37."""
    V, N = 4_800_000, 20_600_000
    counts = _zipf_counts(V, N, 5)
    cdf = frequency_cdf(counts, 0.5).numpy()
    q = np.diff(cdf).astype(np.float64)
    w = counts.double().numpy() + 0.5
    rel = np.abs(q / q.sum() - w / w.sum()) / (w / w.sum())
    assert rel.max() < 2.0 ** -35


def test_invalid_weights_are_refused(lib):
    c, neg, zero = np.array([3, 0, 2], np.int64), np.array([3, -1, 2], np.int64), np.zeros(3, np.int64)
    big = np.array([2 ** 61, 2 ** 61, 1], np.int64)
    cdf = np.zeros(4, np.uint64)
    cases = {"vocab": (c.ctypes.data, 0, 1.0, cdf.ctypes.data),
             "counts": (None, 3, 1.0, cdf.ctypes.data),
             "cdf_out": (c.ctypes.data, 3, 1.0, None),
             "negative count": (neg.ctypes.data, 3, 1.0, cdf.ctypes.data),
             "negative smoothing": (c.ctypes.data, 3, -0.5, cdf.ctypes.data),
             "nan smoothing": (c.ctypes.data, 3, float("nan"), cdf.ctypes.data),
             "inf smoothing": (c.ctypes.data, 3, float("inf"), cdf.ctypes.data),
             "zero weight": (zero.ctypes.data, 3, 0.0, cdf.ctypes.data),
             "above 2^62": (big.ctypes.data, 3, 0.0, cdf.ctypes.data)}
    for what, args in cases.items():
        assert lib.b200kge_frequency_cdf_build(*args) == INVALID, what
        assert lib.b200kge_last_error(), what
    with pytest.raises(ValueError, match="negative"):
        frequency_cdf(torch.tensor([1, -2]), 1.0)
    with pytest.raises(ValueError, match="smoothing"):
        frequency_cdf(torch.tensor([1, 2]), -1.0)
    with pytest.raises(ValueError, match="zero"):
        frequency_cdf(torch.tensor([0, 0]), 0.0)


# ---- the per-entry table of the filtered entry --------------------------------------------------------------------
def _split(E, R, N, seed, heavy=None):
    g = torch.Generator().manual_seed(seed)
    t = torch.stack([torch.randint(0, E, (N,), generator=g), torch.randint(0, R, (N,), generator=g),
                     torch.randint(0, E, (N,), generator=g)], 1)
    extra = [t[:5]]                                               # repeated triples
    if heavy is not None:                                          # (0, 0, ?) with `heavy` objects, (?, 1, 1) alike
        k = torch.arange(heavy)
        extra += [torch.stack([torch.zeros_like(k), torch.zeros_like(k), k], 1),
                  torch.stack([k, torch.ones_like(k), torch.ones_like(k)], 1)]
    return torch.cat([t] + extra)


@pytest.mark.parametrize("slot", [S, P, O])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.5])
def test_below_is_the_brute_force_sum(slot, alpha):
    E, R = 30, 5
    V = R if slot == P else E
    split = _split(E, R, 200, 7 + slot)
    keys, offs, vals, _ = filter_csr(index_KvsAll(split, PAIR[slot]), V)
    cdf = frequency_cdf(torch.bincount(split[:, slot], minlength=V), alpha)
    below, full, first = frequency_below(cdf, offs, vals)
    q = np.diff(cdf.numpy())
    for j in range(len(keys)):
        v = vals[offs[j]:offs[j + 1]].tolist()
        for i, x in enumerate(v):
            # weight of the key's non-positives below x
            want = sum(int(q[y]) for y in range(x) if y not in v[:i])
            assert int(below[offs[j] + i]) == want
    assert np.array_equal(below.numpy().astype(np.uint64), nfq.below_of(cdf.numpy(), offs.numpy(), vals.numpy()))
    assert (full, first) == (0, -1) or alpha == 0


def test_keys_whose_positives_carry_all_the_weight_are_reported():
    """alpha = 0: only ids 2 and 5 have weight; key 1 holds both (full), key 3 holds all ids (full), key 0 holds 2."""
    counts = torch.tensor([0, 0, 4, 0, 0, 1, 0])
    cdf = frequency_cdf(counts, 0.0)
    offs = torch.tensor([0, 1, 4, 5, 12])
    vals = torch.tensor([2, 1, 2, 5, 6] + list(range(7)))
    below, full, first = frequency_below(cdf, offs, vals)
    assert (full, first) == (2, 1)
    _, full, first = frequency_below(frequency_cdf(counts, 1.0), offs, vals)
    assert (full, first) == (1, 3)


def test_invalid_filter_tables_are_refused(lib):
    cdf = np.array([0, 2, 2, 5], np.uint64)
    offs = np.array([0, 2, 3], np.int64)
    vals = np.array([0, 2, 1], np.int64)
    out = np.zeros(3, np.uint64)
    nf, ff = C.c_int64(0), C.c_int64(0)

    def call(cdf=cdf, vocab=3, offs=offs, vals=vals, nk=2, out=out, nf=C.byref(nf), ff=C.byref(ff)):
        ptr = (lambda a: a.ctypes.data if isinstance(a, np.ndarray) else a)
        return lib.b200kge_frequency_filter_build(ptr(cdf), vocab, ptr(offs), ptr(vals), nk, ptr(out), nf, ff)

    assert call() == 0, lib.b200kge_last_error()
    assert out.tolist() == [0, 0, 2]
    bad = {"vocab": dict(vocab=0), "cdf": dict(cdf=None), "offsets": dict(offs=None), "num_keys": dict(nk=-1),
           "values": dict(vals=None), "below_out": dict(out=None), "num_full": dict(nf=None),
           "first_full": dict(ff=None),
           "cdf start": dict(cdf=np.array([1, 2, 2, 5], np.uint64)),
           "cdf decreases": dict(cdf=np.array([0, 3, 2, 5], np.uint64)),
           "cdf zero": dict(cdf=np.zeros(4, np.uint64)),
           "offsets decrease": dict(offs=np.array([0, 3, 2], np.int64), vals=None),
           "value range": dict(vals=np.array([0, 3, 1], np.int64)),
           "values repeat": dict(vals=np.array([2, 2, 1], np.int64)),
           "values descend": dict(vals=np.array([2, 0, 1], np.int64))}
    for what, kw in bad.items():
        assert call(**kw) == INVALID, what
        assert lib.b200kge_last_error(), what


# ---- argument validation of the sampling entries: every buffer is host memory, so an argument that slipped past
# validation would surface as a CUDA error code instead of B200KGE_ERR_INVALID
host_only = pytest.mark.skipif(torch.cuda.is_available(), reason="host buffers only: runs where there is no GPU")
N, K, V, NK = 4, 3, 10, 2
BAD_PLAIN = ("vocab", "n", "K", "out", "cdf")
BAD_FILTERED = ("vocab", "slot", "n", "K", "num_keys", "out", "triples", "keys", "offsets", "values", "cdf", "below")


def _sampling_call(lib, filtered, bad=None):
    keep = [np.zeros(N * 3, np.int64), np.array([0, 1, 0, 2], np.int64), np.array([0, 1, 2], np.int64),
            np.array([3, 4], np.int64), np.zeros(N * K, np.int64), np.arange(V + 1, dtype=np.uint64),
            np.array([3, 3], np.uint64)]
    tri, keys, offs, vals, out, cdf, below = (a.ctypes.data for a in keep)
    a = dict(vocab=V, slot=2, n=N, K=K, num_keys=NK, out=out, triples=tri, keys=keys, offsets=offs, values=vals,
             cdf=cdf, below=below)
    if bad is not None:
        a[bad] = {"vocab": 0, "slot": 3, "n": -1, "K": -1, "num_keys": -1}.get(bad)
    if not filtered:
        return lib.b200kge_sample_frequency(1, 2, a["vocab"], a["cdf"], a["n"], a["K"], a["out"], None)
    return lib.b200kge_sample_frequency_filtered(1, 2, a["vocab"], a["n"], a["K"], a["triples"], a["slot"], a["keys"],
                                                 a["offsets"], a["values"], a["num_keys"], a["cdf"], a["below"],
                                                 a["out"], None)


@host_only
@pytest.mark.parametrize("filtered", [False, True])
def test_valid_sampling_arguments_pass_validation(lib, filtered):
    assert _sampling_call(lib, filtered) != INVALID, lib.b200kge_last_error()


@host_only
@pytest.mark.parametrize("bad", [("plain", b) for b in BAD_PLAIN] + [("filtered", b) for b in BAD_FILTERED],
                         ids=lambda x: f"{x[0]}-{x[1]}")
def test_bad_sampling_argument_is_refused(lib, bad):
    assert _sampling_call(lib, bad[0] == "filtered", bad[1]) == INVALID, lib.b200kge_last_error()


# ---- the mirror ---------------------------------------------------------------------------------------------------
def test_every_id_has_exactly_its_weight_of_preimages():
    """Tiny Q: every t in [0, Q) of the first draw, and every u in [0, Q - M) of the second draw for a key."""
    for counts, alpha in (([3, 0, 1, 0, 5, 2], 0.0), ([3, 0, 1, 0, 5, 2], 1.0), ([0, 0, 0, 0], 1.0)):
        q = [c + int(alpha) for c in counts]             # tiny integer weights: the cdf of q itself
        cdf = nfq.cdf_of(q)
        Q = int(cdf[-1])
        x = nfq.search(cdf, np.arange(Q, dtype=np.uint64))
        assert np.bincount(x, minlength=len(q)).tolist() == q
        V = len(q)
        for v in ([0], [3], [1, 2], [0, 3], [2, 3, 5], list(range(1, V)), list(range(V))):
            v = np.array(sorted(y for y in set(v) if y < V), dtype=np.int64)
            G = nfq.below_of(cdf, [0, len(v)], v)
            rest = int(nfq.rest_of(cdf, v, G))
            assert rest == Q - sum(q[y] for y in v)
            if rest == 0:
                continue
            y = nfq.nonpositive(cdf, v, G, np.arange(rest, dtype=np.uint64))
            want = [0 if i in v else q[i] for i in range(V)]
            assert np.bincount(y, minlength=V).tolist() == want    # no positive, no zero-weight id


@pytest.mark.parametrize("slot", [S, P, O])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 0.5])
def test_mirror_is_the_plain_python_definition(slot, alpha):
    E, R = 20, 4
    V = R if slot == P else E
    split = _split(E, R, 60, 3 + slot, 12 if slot != P else None)
    counts = torch.bincount(split[:, slot], minlength=V)
    cdf = frequency_cdf(counts, alpha).numpy()
    q = np.diff(cdf).tolist()
    keys, offs, vals, _ = filter_csr(index_KvsAll(split, PAIR[slot]), V)
    below = nfq.below_of(cdf, offs.numpy(), vals.numpy())
    tri = torch.cat([split[:30], torch.tensor([[0, 0, 0], [0, 1, 1], [E - 1, R - 1, E - 1]])]).numpy()
    n, K = len(tri), 17
    for seed, offset in ((11, 5), (2 ** 40 + 3, 2 ** 35 + 7)):
        assert np.array_equal(nfq.sample_frequency(n, K, cdf, seed, offset), nfq.plain(n, K, q, seed, offset))
        got = nfq.sample_frequency_filtered(n, K, cdf, seed, offset, tri, slot, keys.numpy(), offs.numpy(),
                                            vals.numpy(), below)
        pos = nfo.positives_of(split, slot)
        assert np.array_equal(got, nfq.plain(n, K, q, seed, offset, tri, slot, pos))


@pytest.mark.parametrize("count", [0, 3])
def test_equal_weights_reproduce_the_uniform_mirrors(count):
    E, R, V = 40, 4, 40
    split = _split(E, R, 200, 9, 25)
    cdf = frequency_cdf(torch.full((V,), count), 1.0 if count == 0 else 0.0).numpy()
    keys, offs, vals, _ = filter_csr(index_KvsAll(split, PAIR[O]), V)
    below = nfq.below_of(cdf, offs.numpy(), vals.numpy())
    tri = split[:64].numpy()
    for seed, offset in ((3, 1), (2 ** 50 + 1, 77)):
        assert np.array_equal(nfq.sample_frequency(64, 33, cdf, seed, offset),
                              nfo.sample_uniform(64, 33, V, seed, offset))
        got = nfq.sample_frequency_filtered(64, 33, cdf, seed, offset, tri, O, keys.numpy(), offs.numpy(),
                                            vals.numpy(), below)
        want = nfo.sample_uniform_filtered(64, 33, V, seed, offset, tri, O, keys.numpy(), offs.numpy(), vals.numpy())
        assert np.array_equal(got, want)


def test_mirror_distribution():
    """10^6 draws, fixed seed: chi-square against q / Q, and a heavy key's filtered draws against the complement."""
    from scipy.stats import chisquare

    V = 50
    counts = torch.from_numpy(np.random.default_rng(2).integers(0, 40, V))
    cdf = frequency_cdf(counts, 0.5).numpy()
    q = np.diff(cdf).astype(np.float64)
    got = nfq.sample_frequency(1000, 1000, cdf, 123, 9)
    assert chisquare(np.bincount(got.reshape(-1), minlength=V), q / q.sum() * got.size).pvalue > 1e-3
    pos = np.sort(np.argsort(-q)[:20])                      # the 20 heaviest ids
    keys, offs = np.array([[0, 0]]), np.array([0, 20])
    below = nfq.below_of(cdf, offs, pos)
    got = nfq.sample_frequency_filtered(1000, 1000, cdf, 123, 9, np.zeros((1000, 3), np.int64), O, keys, offs, pos,
                                        below)
    assert not np.isin(got, pos).any()
    rest = np.setdiff1d(np.arange(V), pos)
    obs = np.bincount(got.reshape(-1), minlength=V)[rest]
    assert chisquare(obs, q[rest] / q[rest].sum() * got.size).pvalue > 1e-3


# ---- job routing ------------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 53, 4, 16


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    sp = ju.synthetic_splits(JE, JR, 150, 20, 20)
    sp["train"] = torch.cat([sp["train"], sp["train"][:10]])       # repeated triples
    return sp


def _job(splits, extra, model="b200_complex", device_sampling=True):
    import jobs_util as ju

    cfg = {"negative_sampling.sampling_type": "frequency", "negative_sampling.num_samples.s": 3,
           "negative_sampling.num_samples.o": 4}
    if device_sampling:
        cfg["user.b200_device_sampling"] = True
    cfg.update(extra)
    job = ju.make_job(model, JE, JR, JD, splits, train_type="negative_sampling", loss="kl", batch_size=32,
                      forward_only=False, extra=cfg, job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    return job


@pytest.fixture()
def mirror(monkeypatch):
    """engine's frequency samplers replaced by the numpy mirror (on CPU tensors); records the calls."""
    calls = []

    def plain(n, K, table, seed, offset):
        calls.append(("plain", offset & 3, None))
        return torch.from_numpy(nfq.sample_frequency(n, K, table.cdf.numpy(), seed, offset))

    def filtered(n, K, table, seed, offset, triples, slot, index):
        calls.append(("filtered", slot, triples.clone()))
        assert index.below_table is table
        return torch.from_numpy(nfq.sample_frequency_filtered(
            n, K, table.cdf.numpy(), seed, offset, triples.numpy(), slot, index.keys.numpy(), index.offsets.numpy(),
            index.values.numpy(), index.below.numpy()))

    def uniform(*a, **kw):
        raise AssertionError("a uniform entry was called for frequency sampling")

    monkeypatch.setattr(engine, "sample_frequency", plain)
    monkeypatch.setattr(engine, "sample_frequency_filtered", filtered)
    monkeypatch.setattr(engine, "sample_uniform", uniform)
    monkeypatch.setattr(engine, "sample_uniform_filtered", uniform)
    return calls


@needs_ref
@pytest.mark.parametrize("alpha", [1, 0, 3])
def test_the_job_constructs_and_keeps_the_weights(splits, alpha, mirror):
    assert not hasattr(torch, "_multinomial_alias_setup")        # KgeFrequencySampler cannot be built here
    job = _job(splits, {"negative_sampling.frequency.smoothing": alpha})
    sm = job._sampler
    assert type(sm).__name__ == "B200FrequencySampler" and job._device_sampling and job._filter_index == {}
    assert sorted(job._frequency) == [S, O]
    for slot in (S, P, O):
        V = JR if slot == P else JE
        want = torch.bincount(splits["train"][:, slot].long(), minlength=V)
        assert torch.equal(sm.counts[slot], want) and sm.smoothing == alpha
    for slot in (S, O):
        assert torch.equal(job._frequency[slot].cdf, frequency_cdf(sm.counts[slot], alpha))
    batch = job._get_collate_fun()(list(range(32)))
    assert batch["negative_samples"] == []                        # the collate draws nothing
    with pytest.raises(NotImplementedError, match="device"):
        sm._sample(batch["triples"], O, 4)
    for slot in (S, O):
        neg = job._device_negatives(32, slot, 0, batch["triples"])
        assert neg.shape == (32, 3 if slot == S else 4)
        assert (neg >= 0).all() and (neg < JE).all()
    assert [c[:2] for c in mirror] == [("plain", S), ("plain", O)]


@needs_ref
@pytest.mark.parametrize("slots,impl", [("o", "standard"), ("so", "fast_if_available"), ("s", "standard")])
def test_filtered_frequency_sampling_takes_the_device_route(splits, slots, impl, mirror):
    extra = {f"negative_sampling.filtering.{c}": True for c in slots}
    extra["negative_sampling.filtering.implementation"] = impl
    job = _job(splits, extra)
    filtered = sorted("spo".index(c) for c in slots)
    assert sorted(job._filter_index) == filtered
    for slot in filtered:
        index = job._filter_index[slot]
        assert index.below_table is job._frequency[slot]
        assert np.array_equal(index.below.numpy().astype(np.uint64),
                              nfq.below_of(job._frequency[slot].cdf.numpy(), index.offsets.numpy(),
                                           index.values.numpy()))
    tri = job._get_collate_fun()(list(range(32)))["triples"]
    for slot in (S, O):
        neg = job._device_negatives(32, slot, 0, tri)
        if slot in filtered:
            pos = nfo.positives_of(splits["train"], slot)
            a, b = nfo.KEY_COLS[slot]
            for i in range(32):
                assert not set(neg[i].tolist()) & pos.get((int(tri[i, a]), int(tri[i, b])), set())
    assert [c[1] for c in mirror if c[0] == "filtered"] == filtered
    assert all(torch.equal(c[2], tri) for c in mirror if c[0] == "filtered")


@needs_ref
def test_fast_filtering_is_refused(splits):
    with pytest.raises(NotImplementedError, match="Use filtering.implementation=standard for this sampler."):
        _job(splits, {"negative_sampling.filtering.o": True, "negative_sampling.filtering.implementation": "fast"})
    job = _job(splits, {"negative_sampling.filtering.implementation": "fast"})     # nothing filtered: served
    assert job._filter_index == {}


@needs_ref
def test_a_key_holding_all_the_weight_is_refused(splits):
    """smoothing 0 and entity 7 the only object of the split: every (s, p) key's positives carry all the O-slot weight."""
    sp = dict(splits)
    tr = sp["train"].clone()
    tr[:, 2] = 7
    sp["train"] = torch.cat([tr, torch.tensor([[2, 1, 7]], dtype=tr.dtype)])
    with pytest.raises(NotImplementedError, match="filtering.o.*all the frequency weight"):
        _job(sp, {"negative_sampling.filtering.o": True, "negative_sampling.frequency.smoothing": 0})
    job = _job(sp, {"negative_sampling.filtering.o": True, "negative_sampling.frequency.smoothing": 1})
    assert sorted(job._filter_index) == [O]


@needs_ref
def test_training_with_a_p_slot_is_refused(splits, mirror):
    job = _job(splits, {"negative_sampling.num_samples.p": 2})
    assert sorted(job._frequency) == [S, P, O]
    job._prepare()
    with pytest.raises(NotImplementedError, match="b200_device_sampling"):
        job.run_epoch()


@needs_ref
def test_without_the_option_the_reference_constructor_runs(splits, mirror):
    """Frequency sampling off the device route is the reference's KgeFrequencySampler, which this torch cannot build;
    shared frequency sampling alike."""
    with pytest.raises(AttributeError, match="_multinomial_alias_setup"):
        _job(splits, {}, device_sampling=False)
    with pytest.raises(AttributeError, match="_multinomial_alias_setup"):
        _job(splits, {"negative_sampling.shared": True})
    assert not mirror
