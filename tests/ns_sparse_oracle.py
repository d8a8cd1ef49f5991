"""TEST INFRASTRUCTURE: the row set of a row-sparse table gradient of one negative-sampling slot (numpy), as LibKGE's
nn.Embedding(sparse=True) produces it: every row the reference looks up for the slot, sorted, whatever its value."""
from __future__ import annotations

import numpy as np


def row_sets(triples, negatives, implementation, num_entities):
    """(entity rows, relation rows) of one slot: the positives' s and o plus every sampled id (`triple`, `batch`), or
    every entity row (`all`, whose open slot goes through embed_all()); the positives' p.  A reciprocal-relations S slot
    is passed as its rewritten triples (o, p + R, s)."""
    tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    neg = np.asarray(negatives, dtype=np.int64).reshape(-1)
    if implementation == "all":
        ent = np.arange(num_entities, dtype=np.int64)
    else:
        ent = np.unique(np.concatenate([tri[:, 0], tri[:, 2], neg]))
    return ent, np.unique(tri[:, 1])
