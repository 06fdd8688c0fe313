"""Pins the CPU statement of the graph range search (tests/graph_range_ref.py): the closure is one set whatever order the worklist
takes, a subset of the exact range search's result with the same distance bytes, equal to it on a complete graph and at radius +inf
on a connected one, monotone in the radius; a row walk stops at its first INVALID, an emptied row contributes nothing, and NaN
distances, ties at the radius and duplicates at radius 0 behave as in the exact statement."""
import numpy as np
import pytest

from tests import datagen, graph_range_ref, range_ref

INVALID = graph_range_ref.INVALID


def _index(oracle, rows, M=8, seed=1):
    ix, _ = oracle.build(rows, M=M, seed=seed)
    g = ix.export()
    return g.points, g.zero, g.upper, g.M


def _segments(offsets, a):
    return [a[int(offsets[i]):int(offsets[i + 1])] for i in range(len(offsets) - 1)]


def _assert_subsequence(got, exact):
    """Every segment of `got` is a subsequence of the same segment of `exact`, with the same distance bytes per id."""
    for gi, gd, ei, ed in zip(_segments(got[0], got[1]), _segments(got[0], got[2]), _segments(exact[0], exact[1]),
                              _segments(exact[0], exact[2])):
        where = {int(p): j for j, p in enumerate(ei)}
        idx = np.array([where[int(p)] for p in gi], dtype=np.int64)
        assert (np.diff(idx) > 0).all() and gd.tobytes() == ed[idx].tobytes()


@pytest.mark.parametrize("order", ["lifo", "reversed", "levels"])
def test_the_closure_does_not_depend_on_the_worklist_order(oracle, order):
    rows, zero, upper, M = _index(oracle, datagen.sift_shaped(700, 12, 1))
    q = datagen.sift_shaped(25, 12, 2)
    full = range_ref.full_order(oracle, rows, q)
    for radius in (float(np.median(full[1][:, 10])), float(np.median(full[1][:, 80]))):
        fifo = graph_range_ref.graph_range_search(oracle, rows, zero, upper, M, q, radius, 20, full=full)
        other = graph_range_ref.graph_range_search(oracle, rows, zero, upper, M, q, radius, 20, order=order, full=full)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(fifo, other))


def test_subset_of_the_exact_range_search_and_monotone_in_the_radius(oracle):
    rows, zero, upper, M = _index(oracle, datagen.sift_shaped(900, 16, 3), M=4)
    q = datagen.sift_shaped(30, 16, 4)
    full = range_ref.full_order(oracle, rows, q)
    prev = None
    for rank in (0, 5, 40, 200, 899):
        radius = float(np.median(full[1][:, rank]))
        got = graph_range_ref.graph_range_search(oracle, rows, zero, upper, M, q, radius, 10, full=full)
        _assert_subsequence(got, range_ref.cut(*full, radius))
        counts = np.diff(got[0])
        if prev is not None:
            assert (counts >= prev).all()
        prev = counts


def test_a_complete_graph_gives_the_exact_result(oracle):
    rows = datagen.uniform(30, 5, 5)
    zero = np.full((30, 32), INVALID, dtype=np.uint32)  # M = 16: every row lists the 29 other points
    for p in range(30):
        zero[p, :29] = [x for x in range(30) if x != p]
    q = datagen.uniform(7, 5, 6)
    full = range_ref.full_order(oracle, rows, q)
    for radius in (float(np.median(full[1][:, 3])), float(np.median(full[1][:, 20])), np.inf):
        got = graph_range_ref.graph_range_search(oracle, rows, zero, [], 16, q, radius, 1, full=full)
        want = range_ref.cut(*full, radius)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))


def test_infinite_radius_on_a_connected_graph_is_every_point(oracle):
    rows, zero, upper, M = _index(oracle, datagen.sift_shaped(500, 8, 7), M=8)
    q = datagen.sift_shaped(10, 8, 8)
    full = range_ref.full_order(oracle, rows, q)
    got = graph_range_ref.graph_range_search(oracle, rows, zero, upper, M, q, np.inf, 5, full=full)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, range_ref.cut(*full, np.inf)))


def test_the_row_walk_stops_at_the_first_invalid():
    zero = np.array([[1, INVALID, 2, 3], [0, INVALID, INVALID, INVALID], [3, INVALID, INVALID, INVALID], [2, INVALID, INVALID, INVALID]],
                    dtype=np.uint32)
    hit = np.ones(4, bool)
    assert graph_range_ref.closure(zero, [0], hit) == {0, 1}  # 2 and 3 sit past row 0's first INVALID
    assert graph_range_ref.closure(zero, [2], hit) == {2, 3}
    assert graph_range_ref.closure(zero, [0, 3], np.array([True, False, True, True])) == {0, 2, 3}


def test_an_emptied_row_contributes_nothing():
    zero = np.array([[INVALID] * 4, [0, 2, INVALID, INVALID], [1, INVALID, INVALID, INVALID]], dtype=np.uint32)
    hit = np.ones(3, bool)
    assert graph_range_ref.closure(zero, [0], hit) == {0}
    assert graph_range_ref.closure(zero, [1], hit) == {0, 1, 2}
    assert graph_range_ref.closure(zero, [1], np.array([True, True, False])) == {0, 1}  # a non-hit is not walked through


def test_nan_ties_and_duplicates(oracle):
    rows = datagen.grid_ties(400, 3, 9, side=4)
    rows[[5, 6]] = rows[4]  # duplicates of row 4
    rows[10, 1] = np.nan     # NaN distance to every query
    zero = np.full((400, 8), INVALID, dtype=np.uint32)
    ring = np.arange(400, dtype=np.uint32)
    zero[:, 0], zero[:, 1] = np.roll(ring, 1), np.roll(ring, -1)  # a ring: connected, every row reaches every other
    q = rows[[4, 0]].copy()
    full = range_ref.full_order(oracle, rows, q)
    for radius in (0.0, 1.0, 2.0, np.inf):
        got = graph_range_ref.graph_range_search(oracle, rows, zero, [], 4, q, radius, 4, full=full)
        exact = range_ref.cut(*full, radius)
        _assert_subsequence(got, exact)
        assert not np.isin(got[1], [10]).any()  # NaN is never a hit
    # ef = n: nearest(q) holds every point, so radius 0 finds exactly the copies of the query's row, in PointId order
    got = graph_range_ref.graph_range_search(oracle, rows, zero, [], 4, q[:1], 0.0, 400, full=(full[0][:1], full[1][:1]))
    copies = np.flatnonzero((rows == q[0]).all(1))
    assert {4, 5, 6} <= set(copies.tolist()) and got[1].tolist() == copies.tolist() and (got[2] == 0).all()
    got = graph_range_ref.graph_range_search(oracle, rows, zero, [], 4, q, np.inf, 4, full=full)
    assert (np.diff(got[0]) == 399).all()  # the ring reaches every row but the NaN one
    got = graph_range_ref.graph_range_search(oracle, rows, zero, [], 4, q, -1.0, 4, full=full)
    assert (got[0] == 0).all()
