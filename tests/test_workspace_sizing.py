"""CPU tests of the training workspace sizes (host code, no device): b200kge_train_1vsall_workspace_bytes and
b200kge_ns_backward_workspace_bytes return, on a grid of shapes for every model, the sizes the per-variant sizing
functions they replace returned (values pinned below), so no caller's allocation shrinks."""
import pytest

# (model, n, E, D, workspace_bytes, 1vsAll backward, 1vsAll dropout, 1vsAll reciprocal, NS backward, NS dropout): the
# last six are the values of b200kge_workspace_bytes(model, n, E, D, 0), the former
# b200kge_train_1vsall_{backward,dropout,reciprocal}_workspace_bytes, the NS backward's former Python-side size
# n * (D + 32) * 4 + 1024 and the former b200kge_ns_dropout_workspace_bytes
PINNED = [
    (0, 0, 100, 16, 36624, 60704, 86048, 86304, 1024, 0),
    (0, 7, 1000, 64, 371480, 1404976, 1809644, 1809956, 3712, 9216),
    (0, 512, 14541, 200, 24432820, 240609064, 195600744, 240609064, 476160, 2109440),
    (1, 0, 100, 16, 36624, 60704, 86048, 86304, 1024, 0),
    (1, 7, 1000, 64, 371480, 1404976, 1809644, 1809956, 3712, 9216),
    (1, 512, 14541, 200, 24432820, 240609064, 195600744, 240609064, 476160, 2109440),
    (2, 0, 100, 16, 36624, 60704, 86048, 86304, 1024, 0),
    (2, 7, 1000, 64, 371480, 1404976, 1809644, 1809956, 3712, 9216),
    (2, 512, 14541, 200, 24432820, 240609064, 195600744, 240609064, 476160, 2109440),
    (3, 0, 100, 16, 36624, 53344, 78688, 78944, 1024, 0),
    (3, 7, 1000, 64, 371480, 1122864, 1532140, 1532452, 3712, 7680),
    (3, 512, 14541, 200, 24432820, 216888584, 173584200, 216888584, 476160, 1699840),
    (4, 0, 100, 16, 36624, 60704, 86048, 86304, 1024, 0),
    (4, 7, 1000, 64, 371480, 1404976, 2035436, 2035748, 3712, 235008),
    (4, 512, 14541, 200, 24432820, 240609064, 358621544, 358625896, 476160, 165130240),
    (5, 0, 100, 16, 36624, 40720, 61968, 62224, 1024, 0),
    (5, 7, 1000, 64, 371480, 622968, 999256, 999568, 3712, 9216),
    (5, 512, 14541, 200, 24432820, 264552628, 140602100, 264552628, 476160, 2109440),
    (6, 0, 100, 16, 36624, 40720, 61968, 62224, 1024, 0),
    (6, 7, 1000, 64, 371480, 622968, 997464, 997776, 3712, 7680),
    (6, 512, 14541, 200, 24432820, 264552628, 140192500, 264552628, 476160, 1699840),
]


@pytest.fixture(scope="module")
def lib():
    from kge_b200.build import build_native
    from kge_b200 import _lib

    build_native()
    return _lib.load()


@pytest.mark.parametrize("row", PINNED, ids=lambda r: "m{}-n{}-E{}-D{}".format(*r[:4]))
def test_train_1vsall_workspace_bytes(lib, row):
    model, n, E, D, fwd, bwd, drop, recip = row[:8]
    assert lib.b200kge_workspace_bytes(model, n, E, D, 0) == fwd
    plain = lib.b200kge_train_1vsall_workspace_bytes(model, n, E, D, 0)
    dropout = lib.b200kge_train_1vsall_workspace_bytes(model, n, E, D, 1)
    assert plain == max(fwd, bwd)
    assert dropout == drop + n * 8 + 256        # + the reciprocal step's p + R index
    assert max(plain, dropout) == recip


@pytest.mark.parametrize("row", PINNED, ids=lambda r: "m{}-n{}-E{}-D{}".format(*r[:4]))
def test_ns_backward_workspace_bytes(lib, row):
    model, n, E, D = row[:4]
    ns_plain, ns_drop = row[8:]
    for K in (1, 30):       # K does not enter the size
        assert lib.b200kge_ns_backward_workspace_bytes(model, n, K, D, 0) == ns_plain
        assert lib.b200kge_ns_backward_workspace_bytes(model, n, K, D, 1) == ns_drop
