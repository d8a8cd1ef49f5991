"""Filtered negative sampling on the CPU: the numpy mirror of b200kge_sample_uniform_filtered (tests/ns_filter_oracle.py)
pinned against the plain-Python Philox and the brute-force definition, the host filter-index builder against a
dict-of-sets, and the negative-sampling job's routing of `negative_sampling.filtering.*` with
`user.b200_device_sampling`.  The kernel is checked against the same mirror in tests/test_gpu_ns_filter.py."""
import numpy as np
import pytest
import torch

import ns_filter_oracle as nfo
import philox_ref
from kge_b200 import engine, hostenv
from kge_b200.indexing import filter_csr, index_KvsAll

S, P, O = 0, 1, 2
PAIR = {S: "po", P: "so", O: "sp"}


# ---- the mirror -------------------------------------------------------------------------------------------------------
def test_umulhi_is_the_high_word_of_the_product():
    g = np.random.default_rng(1)
    a = g.integers(0, 2 ** 63, 1000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    b = g.integers(1, 2 ** 40, 1000, dtype=np.uint64)
    got = nfo.umulhi(a, b)
    assert [int(x) for x in got] == [(int(x) * int(y)) >> 64 for x, y in zip(a, b)]


@pytest.mark.parametrize("n,K,vocab,seed,offset", [(3, 7, 40943, 5, 1), (2, 9, 11, 2 ** 40 + 3, 2 ** 35 + 7),
                                                   (1, 1, 1, 0, 0)])
def test_first_draw_is_sample_uniform(n, K, vocab, seed, offset):
    assert nfo.sample_uniform(n, K, vocab, seed, offset).reshape(-1).tolist() == \
        philox_ref.sample_uniform(n, K, vocab, seed, offset)


def test_second_draw_uses_the_high_counter_domain():
    seed, offset = 2 ** 33 + 9, 77
    for e in (0, 1, 6, 13):
        block = (e // 2) | (1 << 63)
        c = philox_ref.philox4x32_10([block & 0xFFFFFFFF, block >> 32, offset & 0xFFFFFFFF, offset >> 32],
                                     (seed & 0xFFFFFFFF, seed >> 32))
        want = (c[1] << 32 | c[0]) if e % 2 == 0 else (c[3] << 32 | c[2])
        assert int(nfo.words(np.array([e]), seed, offset, nfo.FILTER_DOMAIN)[0]) == want
        assert want != int(nfo.words(np.array([e]), seed, offset)[0])


def _split(E, R, N, seed, heavy=None):
    g = torch.Generator().manual_seed(seed)
    t = torch.stack([torch.randint(0, E, (N,), generator=g), torch.randint(0, R, (N,), generator=g),
                     torch.randint(0, E, (N,), generator=g)], 1)
    extra = [t[:5]]                                               # repeated triples
    if heavy is not None:                                          # (s, p, ?) with `heavy` objects, (?, p, o) alike
        k = torch.arange(heavy)
        extra += [torch.stack([torch.zeros_like(k), torch.zeros_like(k), k], 1),
                  torch.stack([k, torch.ones_like(k), torch.ones_like(k)], 1)]
    return torch.cat([t] + extra)


@pytest.mark.parametrize("slot", [S, P, O])
@pytest.mark.parametrize("heavy", [None, 19, 20])
def test_mirror_is_the_brute_force_definition(slot, heavy):
    """All three slots; keys with few positives, an absent key, m = V - 1 and m = V (rows of -1)."""
    E, R = 20, 4
    V = R if slot == P else E
    split = _split(E, R, 60, 3 + slot, heavy if slot != P else None)
    keys, offs, vals, mx = filter_csr(index_KvsAll(split, PAIR[slot]), V)
    # rows of the heavy (s, p) = (0, 0) and (p, o) = (1, 1) keys, and of a key absent from the split
    tri = torch.cat([split[:40], torch.tensor([[0, 0, 0], [0, 1, 1], [E - 1, R - 1, E - 1]])]).numpy()
    n, K = len(tri), 23
    got = nfo.sample_uniform_filtered(n, K, V, 11, 5, tri, slot, keys.numpy(), offs.numpy(), vals.numpy())
    pos = nfo.positives_of(split, slot)
    want = nfo.brute_force(n, K, V, 11, 5, tri, slot, pos)
    assert np.array_equal(got, want)
    a, b = nfo.KEY_COLS[slot]
    sizes = []
    for i in range(n):
        p = pos.get((int(tri[i, a]), int(tri[i, b])), set())
        sizes.append(len(p))
        if len(p) >= V:
            assert (got[i] == -1).all()
        else:
            assert (got[i] >= 0).all() and (got[i] < V).all() and not set(got[i].tolist()) & p
    assert mx == max(len(p) for p in pos.values())
    if heavy is not None and slot != P:
        assert max(sizes) >= heavy                       # the m = V - 1 / m = V rows were exercised


def test_mirror_distribution_over_the_non_positives():
    """V = 50, m = 30, 10^6 draws: chi-square over the 20 non-positives, fixed seed (p-value far from 0)."""
    from scipy.stats import chisquare

    V, m = 50, 30
    pos = np.sort(np.random.default_rng(0).choice(V, m, replace=False))
    keys, offs = np.array([[0, 0]]), np.array([0, m])
    tri = np.zeros((1000, 3), dtype=np.int64)
    got = nfo.sample_uniform_filtered(1000, 1000, V, 123, 9, tri, O, keys, offs, pos)
    assert not np.isin(got, pos).any()
    counts = np.bincount(got.reshape(-1), minlength=V)[np.setdiff1d(np.arange(V), pos)]
    assert chisquare(counts).pvalue > 1e-3


# ---- the index builder ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slot", [S, P, O])
def test_filter_csr_is_the_dict_of_sets(slot):
    E, R = 30, 5
    split = _split(E, R, 200, 7 + slot)
    keys, offs, vals, mx = filter_csr(index_KvsAll(split, PAIR[slot]), R if slot == P else E)
    want = nfo.positives_of(split, slot)
    got = {(int(a), int(b)): vals[offs[j]:offs[j + 1]].tolist() for j, (a, b) in enumerate(keys.tolist())}
    assert sorted(got) == sorted(want) and keys.tolist() == sorted(keys.tolist())
    for k, v in got.items():
        assert v == sorted(want[k])                    # sorted, duplicates removed
    assert mx == max(len(v) for v in want.values())


def test_filter_csr_of_unsorted_and_repeated_keys():
    class Index:
        _keys = torch.tensor([[3, 1], [0, 2], [3, 1]], dtype=torch.int32)
        _values_offset = torch.tensor([0, 3, 4, 6], dtype=torch.int32)
        _values = torch.tensor([5, 1, 5, 7, 2, 1], dtype=torch.int32)

    keys, offs, vals, mx = filter_csr(Index(), 8)
    assert keys.tolist() == [[0, 2], [3, 1]] and offs.tolist() == [0, 1, 4] and vals.tolist() == [7, 1, 2, 5]
    assert mx == 3
    with pytest.raises(ValueError, match="outside"):
        filter_csr(Index(), 7)
    Index._values_offset = torch.tensor([0, 3, 2, 6], dtype=torch.int32)
    with pytest.raises(ValueError, match="decrease"):
        filter_csr(Index(), 8)


def test_filter_csr_of_an_empty_index():
    keys, offs, vals, mx = filter_csr(index_KvsAll(torch.zeros((0, 3), dtype=torch.int64), "sp"), 5)
    assert keys.shape == (0, 2) and offs.tolist() == [0] and vals.numel() == 0 and mx == 0


# ---- job routing ------------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
JE, JR, JD = 53, 4, 16


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    sp = ju.synthetic_splits(JE, JR, 150, 20, 20)
    sp["train"] = torch.cat([sp["train"], sp["train"][:10]])       # repeated triples
    return sp


def _job(splits, extra, model="b200_complex"):
    import jobs_util as ju

    cfg = {"negative_sampling.num_samples.s": 3, "negative_sampling.num_samples.o": 4}
    cfg.update(extra)
    job = ju.make_job(model, JE, JR, JD, splits, train_type="negative_sampling", loss="kl", batch_size=32,
                      forward_only=False, extra=cfg, job_class="B200TrainingJobNegativeSampling")
    job.epoch += 1
    return job


@pytest.fixture()
def mirror(monkeypatch):
    """engine's samplers replaced by the numpy mirror (on CPU tensors); records the filtered calls."""
    calls = []

    def filtered(n, K, vocab, seed, offset, triples, slot, index):
        calls.append((slot, triples.clone()))
        out = nfo.sample_uniform_filtered(n, K, vocab, seed, offset, triples.numpy(), slot, index.keys.numpy(),
                                          index.offsets.numpy(), index.values.numpy())
        return torch.from_numpy(out)

    monkeypatch.setattr(engine, "sample_uniform_filtered", filtered)
    monkeypatch.setattr(engine, "sample_uniform",
                        lambda n, K, vocab, seed, offset, device: torch.from_numpy(
                            nfo.sample_uniform(n, K, vocab, seed, offset)))
    return calls


@needs_ref
@pytest.mark.parametrize("slots,split", [("o", ""), ("s", ""), ("so", ""), ("so", "valid")])
def test_filtering_with_device_sampling_takes_the_device_route(splits, slots, split, mirror):
    extra = {"user.b200_device_sampling": True, "negative_sampling.filtering.split": split}
    extra.update({f"negative_sampling.filtering.{c}": True for c in slots})
    job = _job(splits, extra)
    filtered = sorted("spo".index(c) for c in slots)
    assert job._device_sampling and sorted(job._filter_index) == filtered
    fsplit = split or "train"
    for slot in filtered:
        # the job's index is the dict-of-sets of the filtering split, from the reference's dataset.index
        index = job._filter_index[slot]
        want = nfo.positives_of(splits[fsplit], slot)
        got = {(a, b): index.values[index.offsets[j]:index.offsets[j + 1]].tolist()
               for j, (a, b) in enumerate(index.keys.tolist())}
        assert got == {k: sorted(v) for k, v in want.items()}
    batch = job._get_collate_fun()(list(range(32)))
    assert batch["negative_samples"] == []                        # the collate draws nothing
    tri = batch["triples"]
    for slot in (S, O):
        neg = job._device_negatives(32, slot, 0, tri)
        assert neg.shape == (32, 3 if slot == S else 4)
        if slot in filtered:
            pos = nfo.positives_of(splits[fsplit], slot)
            a, b = nfo.KEY_COLS[slot]
            for i in range(32):
                assert not set(neg[i].tolist()) & pos.get((int(tri[i, a]), int(tri[i, b])), set())
    assert [c[0] for c in mirror] == filtered
    assert all(torch.equal(c[1], tri) for c in mirror)


@needs_ref
def test_reciprocal_wrapper_filters_the_s_slot_on_the_dataset_triples(splits, mirror):
    import jobs_util as ju

    cfg = {"reciprocal_relations_model.base_model.type": "b200_complex", "user.b200_device_sampling": True,
           "negative_sampling.filtering.s": True, "negative_sampling.num_samples.s": 3,
           "negative_sampling.num_samples.o": 4}
    job = ju.make_job("reciprocal_relations_model", JE, JR, JD, splits, train_type="negative_sampling", loss="kl",
                      batch_size=32, forward_only=False, imports=("b200_complex",), extra=cfg,
                      job_class="B200TrainingJobNegativeSampling")
    assert sorted(job._filter_index) == [S]
    idx = job._filter_index[S]
    assert idx.vocab == JE and int(idx.keys[:, 0].max()) < JR      # keys (p, o) with the dataset's relation ids
    tri = job._get_collate_fun()(list(range(32)))["triples"]
    job._device_negatives(32, S, 0, tri)
    assert torch.equal(mirror[0][1], tri)


@needs_ref
def test_a_key_covering_the_vocabulary_is_refused_at_setup(splits):
    sp = dict(splits)
    k = torch.arange(JE, dtype=sp["train"].dtype)
    sp["train"] = torch.cat([sp["train"], torch.stack([torch.full_like(k, 2), torch.full_like(k, 1), k], 1)])
    with pytest.raises(NotImplementedError, match="filtering.o"):
        _job(sp, {"user.b200_device_sampling": True, "negative_sampling.filtering.o": True})
    job = _job(sp, {"user.b200_device_sampling": True, "negative_sampling.filtering.s": True})   # (p, o) keys are fine
    assert sorted(job._filter_index) == [S]


@needs_ref
def test_training_with_a_filtered_p_slot_is_refused(splits, mirror):
    """The device route serves no P-slot training step, as with unfiltered device sampling: the job refuses it rather
    than train on the host route, which it did before the filtered route existed."""
    job = _job(splits, {"user.b200_device_sampling": True, "negative_sampling.num_samples.p": 2,
                        "negative_sampling.filtering.p": True})
    assert sorted(job._filter_index) == [P]
    job._prepare()
    with pytest.raises(NotImplementedError, match="b200_device_sampling"):
        job.run_epoch()


@needs_ref
def test_filtering_without_the_option_takes_the_host_route(splits, mirror):
    job = _job(splits, {"negative_sampling.filtering.o": True, "negative_sampling.implementation": "triple"})
    assert not job._device_sampling and job._filter_index == {}
    batch = job._get_collate_fun()(list(range(32)))
    neg = batch["negative_samples"][O].samples()                 # the reference sampler drew and filtered them
    pos = nfo.positives_of(splits["train"], O)
    tri = batch["triples"]
    for i in range(32):
        assert not set(neg[i].tolist()) & pos.get((int(tri[i, 0]), int(tri[i, 1])), set())
    assert not mirror
