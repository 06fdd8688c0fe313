"""Pins the CPU statement of the range search (tests/range_ref.py) on small cases an independent numpy computation can check: ties
at the radius are included, NaN distances never are, a cosine index compares the reported 1 - cos with the radius, and the hits are
a prefix of the full exact ordering."""
import numpy as np

from tests import cosine_ref, datagen, range_ref


def _pairwise(rows, q):
    """Squared L2 of integer-valued rows: every sum is an exact small integer in f32, so any order gives the same bits."""
    return ((q[:, None, :].astype(np.float64) - rows[None, :, :]) ** 2).sum(-1).astype(np.float32)


def _segments(offsets, a):
    return [a[int(offsets[i]):int(offsets[i + 1])] for i in range(len(offsets) - 1)]


def test_ties_at_the_radius_are_included(oracle):
    rows = datagen.grid_ties(600, 3, 1, side=5)
    q = datagen.grid_ties(12, 3, 2, side=5)
    d = _pairwise(rows, q)
    for radius in (0.0, 1.0, 2.0, 5.0, 6.0):
        offsets, ids, dist = range_ref.range_search(oracle, rows, q, radius)
        for i, (si, sd) in enumerate(zip(_segments(offsets, ids), _segments(offsets, dist))):
            want = np.flatnonzero(d[i] <= radius)
            want = want[np.lexsort((want, d[i][want]))]  # by distance, then PointId
            assert (si == want).all() and sd.tobytes() == d[i][want].tobytes()
            assert (d[i][si] == radius).sum() == (d[i] == radius).sum()  # every row at exactly the radius


def test_radius_zero_finds_duplicates_and_a_negative_radius_nothing(oracle):
    rows = datagen.grid_ties(300, 2, 3, side=4)
    q = rows[[0, 17, 299]]
    offsets, ids, _ = range_ref.range_search(oracle, rows, q, 0.0)
    for i, seg in enumerate(_segments(offsets, ids)):
        assert (seg == np.flatnonzero((rows == q[i]).all(1))).all()
    offsets, ids, dist = range_ref.range_search(oracle, rows, q, -1e-30)
    assert (offsets == 0).all() and ids.size == 0 and dist.size == 0


def test_nan_never_matches(oracle):
    rows = datagen.uniform(200, 6, 4)
    rows[[3, 150], 2] = np.nan
    q = datagen.uniform(5, 6, 5)
    q[4, 0] = np.nan  # every distance NaN
    offsets, ids, dist = range_ref.range_search(oracle, rows, q, np.inf)
    counts = np.diff(offsets)
    assert (counts[:4] == 198).all() and counts[4] == 0
    assert not np.isin(ids, [3, 150]).any() and not np.isnan(dist).any()


def test_inf_radius_keeps_infinite_distances(oracle):
    rows = datagen.uniform(50, 4, 6)
    rows[7] = 1e20  # the squared distance overflows to +inf
    q = datagen.uniform(3, 4, 7)
    offsets, ids, dist = range_ref.range_search(oracle, rows, q, np.inf)
    assert (np.diff(offsets) == 50).all()
    assert (ids.reshape(3, 50)[:, -1] == 7).all() and np.isinf(dist.reshape(3, 50)[:, -1]).all()
    offsets, _, _ = range_ref.range_search(oracle, rows, q, np.finfo(np.float32).max)
    assert (np.diff(offsets) == 49).all()


def test_cosine_compares_the_reported_distance(oracle):
    rows = cosine_ref.normalize(oracle, datagen.uniform(400, 8, 8) - 0.5)
    q = datagen.uniform(6, 8, 9) - 0.5
    ids, d = oracle.bruteforce(rows, cosine_ref.normalize(oracle, q), 400)  # squared L2 of the unit rows = 2 (1 - cos)
    radius = float(cosine_ref.reported(d)[:, 40].min())
    offsets, got_ids, got_dist = range_ref.range_search(oracle, rows, q, radius, metric="cosine")
    reported = cosine_ref.reported(d)
    assert (np.diff(offsets) == (reported <= radius).sum(1)).all()
    assert (np.diff(offsets) > (d <= radius).sum(1)).all()  # comparing the squared L2 itself would keep fewer
    assert got_dist.tobytes() == np.concatenate([reported[i, :c] for i, c in enumerate(np.diff(offsets))]).tobytes()


def test_prefix_of_the_full_ordering_and_monotone_in_the_radius(oracle):
    rows = datagen.sift_shaped(500, 16, 10)
    q = datagen.sift_shaped(9, 16, 11)
    ids, dist = oracle.bruteforce(rows, q, 500)
    prev = None
    for radius in sorted(float(x) for x in dist[:, [0, 5, 50, 499]].ravel()):
        offsets, got, _ = range_ref.range_search(oracle, rows, q, radius)
        counts = np.diff(offsets)
        for i, seg in enumerate(_segments(offsets, got)):
            assert (seg == ids[i, :counts[i]]).all()
            assert counts[i] == 500 or dist[i, counts[i]] > radius
        if prev is not None:
            assert (counts >= prev).all()
        prev = counts


def test_id_map_applies_after_ordering(oracle):
    rows = np.zeros((10, 2), np.float32)  # all tied
    gmap = np.arange(10, dtype=np.uint32)[::-1] + 100
    offsets, ids, _ = range_ref.range_search(oracle, rows, rows[:1], 0.0, id_map=gmap)
    assert offsets[-1] == 10 and (ids == gmap).all()  # PointId order, not the mapped ids' order


def test_empty_rows():
    offsets, ids, dist = range_ref.cut(np.zeros((4, 0), np.uint32), np.zeros((4, 0), np.float32), 1.0)
    assert (offsets == 0).all() and offsets.shape == (5,) and ids.size == 0 and dist.size == 0
