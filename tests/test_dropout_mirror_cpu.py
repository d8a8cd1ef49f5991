"""The vectorised mask mirror (tests/philox_np.py) against the scalar one (tests/philox_ref.py, tests/dropout_oracle.py):
the raw Philox4x32-10 words on random and extreme counters and keys, and the keep masks bit for bit at row widths that
make blocks straddle rows, at rates from 0 to 0.999 and at element indexes up to just below the 2^48 limit, where the
high counter word carries group bits as well as the stream."""
import numpy as np
import pytest
import torch

import dropout_oracle as dro
import philox_np
from philox_ref import MASK, philox4x32_10

ONES = MASK


def _words(counter, key):
    c = philox_np.philox4x32_10(*(np.array([x], dtype=np.uint64) for x in counter), key)
    return [int(w[0]) for w in c]


def test_philox_words_match_the_scalar_reference():
    rng = np.random.default_rng(0)
    cases = [([0, 0, 0, 0], (0, 0)), ([ONES] * 4, (ONES, ONES)), ([ONES, 0, ONES, 0], (0, ONES)),
             ([1, 2, 3, 4], (5, 6))]
    cases += [([int(x) for x in rng.integers(0, 2 ** 32, 4, dtype=np.uint64)],
               tuple(int(x) for x in rng.integers(0, 2 ** 32, 2, dtype=np.uint64))) for _ in range(64)]
    for counter, key in cases:
        assert _words(counter, key) == philox4x32_10(counter, key), (counter, key)


def test_philox_words_vectorised_over_counters():
    rng = np.random.default_rng(1)
    c = [rng.integers(0, 2 ** 32, 257, dtype=np.uint64) for _ in range(4)]
    key = (0xDEADBEEF, ONES)
    got = philox_np.philox4x32_10(*c, key)
    for i in range(257):
        assert [int(w[i]) for w in got] == philox4x32_10([int(x[i]) for x in c], key)


# element indexes row_base * dim around 2^32, 2^34 and just below 2^48 (with odd row_base: blocks straddle rows)
def _base(target, dim):
    rb = target // dim
    return rb | 1


@pytest.mark.parametrize("dim", [5, 35, 66, 512])
@pytest.mark.parametrize("p", [0.0, 1e-7, 0.3, 0.999])
@pytest.mark.parametrize("seed,call,stream,target", [
    (0, 0, 0, 0), (2 ** 32 + 7, 2 ** 32 + 1, 3, 2 ** 32), (2 ** 63 + 5, 2 ** 40 + 9, 17, 2 ** 34),
    (ONES, 2 ** 64 - 1, 23, 2 ** 48 - 2 ** 12)])
def test_mask_matches_the_scalar_mirror(dim, p, seed, call, stream, target):
    rows = max(1, 64 // dim + 2)
    rb = _base(target, dim) if target else 3
    if (rb + rows) * dim > 2 ** 48:
        rb = 2 ** 48 // dim - rows
    got = philox_np.mask(p, seed, call, stream, rows, dim, rb)
    assert got.dtype == torch.bool and got.shape == (rows, dim)
    assert torch.equal(got, dro.mask(p, seed, call, stream, rows, dim, rb))


def test_mask_at_the_last_element_below_2_48():
    dim = 66
    rb = 2 ** 48 // dim - 2
    for rows in (1, 2):
        assert torch.equal(philox_np.mask(0.5, 11, 2 ** 33, 5, rows, dim, rb),
                           dro.mask(0.5, 11, 2 ** 33, 5, rows, dim, rb))
    rb = (2 ** 48 - 4) // 4                                    # dim 4: the final element is 2^48 - 1
    assert torch.equal(philox_np.mask(0.5, 1, 2, 3, 1, 4, rb), dro.mask(0.5, 1, 2, 3, 1, 4, rb))


def test_empty_and_keep_all():
    assert philox_np.mask(0.3, 1, 2, 0, 0, 5).shape == (0, 5)
    assert philox_np.mask(0.3, 1, 2, 0, 4, 0).shape == (4, 0)
    assert bool(philox_np.mask(0.0, 1, 2, 0, 9, 7, 5).all())


def test_keep_rate_at_table_scale():
    m = philox_np.mask(0.4, 2024, 77, 2, 14541, 512)
    assert abs(float(m.float().mean()) - 0.6) < 2e-3
    # rows differ and so do draws: no accidental reuse of counters across rows or streams
    assert not torch.equal(m[0], m[1])
    assert not torch.equal(m[:64], philox_np.mask(0.4, 2024, 77, 3, 64, 512))
