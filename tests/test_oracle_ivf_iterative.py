"""The restatement of ivfflat.iterative_scan on the CPU oracle (tests/ivf_iter_oracle.py) against the reference's regression output
for the iterative section of test/sql/ivfflat_vector.sql (test/expected/ivfflat_vector.out:93-128)."""
import numpy as np
import pytest

import oracle as O
from tests.ivf_iter_oracle import iter_scan

ROWS = np.array([[0, 0, 0], [1, 2, 3], [1, 1, 1]], dtype=np.float32)
QUERY = np.array([3, 3, 3], dtype=np.float32)
MAX_LISTS = 32768   # IVFFLAT_MAX_LISTS, the default of ivfflat.max_probes


def three_lists(rows):
    """lists = 3 with the rows as centres: one row per list, ids = row numbers"""
    offsets = np.arange(len(rows) + 1, dtype=np.int64) if len(rows) else np.zeros(4, dtype=np.int64)
    return O.Ivf(O.VECTOR, O.L2_SQUARED, ROWS, offsets, rows.reshape(-1, 3), np.arange(len(rows), dtype=np.int64), dim=3)


def returned(ix, max_probes):
    return [ROWS[i].tolist() for ids, _ in iter_scan(ix, QUERY, 1, max_probes) for i in ids]


@pytest.fixture(autouse=True)
def total_order():
    O.ivf_set_tie_mode(True)
    yield
    O.ivf_set_tie_mode(False)


def test_default_max_probes_returns_every_row_group_by_group():
    assert returned(three_lists(ROWS), MAX_LISTS) == [[1, 2, 3], [1, 1, 1], [0, 0, 0]]


@pytest.mark.parametrize("max_probes,want", [(1, [[1, 2, 3]]), (2, [[1, 2, 3], [1, 1, 1]])])
def test_max_probes_bounds_the_lists_scanned(max_probes, want):
    assert returned(three_lists(ROWS), max_probes) == want


def test_empty_index_returns_no_rows():
    ix = three_lists(np.zeros((0, 3), dtype=np.float32))
    groups = iter_scan(ix, QUERY, 1, MAX_LISTS)
    assert len(groups) == 3 and all(len(ids) == 0 for ids, _ in groups)


def test_groups_are_sorted_scans_of_consecutive_probe_lists():
    rng = np.random.default_rng(7)
    centers = rng.standard_normal((12, 8)).astype(np.float32)
    rows = rng.standard_normal((600, 8)).astype(np.float32)
    assign = O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers)
    order = np.argsort(assign, kind="stable")
    offsets = np.zeros(13, dtype=np.int64)
    offsets[1:] = np.cumsum(np.bincount(assign, minlength=12))
    ix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, offsets, rows[order], order.astype(np.int64))
    q = rng.standard_normal(8).astype(np.float32)
    lists, _ = ix.scan_lists(q, 7)
    groups = iter_scan(ix, q, 3, 7)
    assert [len(ids) for ids, _ in groups] == [int(sum(offsets[l + 1] - offsets[l] for l in lists[g:g + 3])) for g in (0, 3, 6)]
    for g, (ids, dist) in zip((0, 3, 6), groups):
        assert np.all(np.diff(dist) >= 0)
        want = set(int(order[r]) for l in lists[g:g + 3] for r in range(offsets[l], offsets[l + 1]))
        assert set(ids.tolist()) == want
    # max_probes below probes is raised to probes (iterative_scan = off): one group
    assert len(iter_scan(ix, q, 3, 1)) == 1
