"""The CPU statement of the index insert (tests/insert_statement.py, statements/insert_statement.cpp) checked on its own.

tests/test_gpu_insert.py compares GPU inserts with this statement bit for bit, so the statement is anchored here:
  * its batched build is oracle.build_batched (the two share no code: the statement states the batch body once, for the build and
    the insert);
  * a build stopped at a layer-0 batch boundary n0, then given the rows [n0, n) by the insert, is the full batched build, for every
    schedule, heuristic and simple selection, f32 and cosine rows;
  * with one insert per batch the insert is the sequential Construction::insert order (oracle.build);
  * the recall an insert gives up against a full build (the upper layers keep sampling the first n0 points) is measured here, and
    the GPU test holds the GPU's graph to the same bound.
"""
import numpy as np
import pytest

from tests import cosine_ref, datagen
from tests import insert_statement as S


def _same(ga, gb):
    assert ga.points.shape == gb.points.shape and ga.points.tobytes() == gb.points.tobytes()
    bad = np.nonzero((ga.zero != gb.zero).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} zero rows differ, first pid {bad[0]}: {ga.zero[bad[0]][:12]} vs {gb.zero[bad[0]][:12]}"
    assert len(ga.upper) == len(gb.upper)
    for x, y in zip(ga.upper, gb.upper):
        assert x.shape == y.shape and (x == y).all()


def layer0_boundaries(oracle, n, M, max_batch, growth):
    """The PointIds where a layer-0 batch of the batched build begins (build.cu's schedule; layer 0 starts at n_1)."""
    counts = oracle.layer_schedule(n, M)
    g0 = max(counts[1] if len(counts) > 1 else 1, 1)
    out = []
    while g0 < n:
        out.append(g0)
        g0 += min(min(max_batch, max(1, g0 // growth)), n - g0)
    return out


def test_statement_build_is_the_oracle_batched_build(oracle):
    rows = datagen.uniform(1500, 16, 3)
    for kw in ({}, {"heuristic": 0}, {"M": 8, "keep_pruned": 0}):
        for mb, gr in ((16384, 8), (7, 8), (1, 8)):
            g, ids = S.build_batched(rows, mb, gr, threads=4, **kw)
            ref, ids_ref, _ = oracle.build_batched(rows, mb, gr, threads=4, **kw)
            assert (ids == ids_ref).all()
            _same(g, ref.export())


CONTINUATION = [
    # (data, n, dim, params, insert_batch)
    ("uniform", 1500, 16, {}, 0),
    ("uniform", 1500, 16, {}, 1),
    ("uniform", 1500, 16, {}, 7),
    ("uniform", 1500, 16, {}, 64),
    ("uniform", 1500, 16, {"heuristic": 0}, 0),
    ("uniform", 1500, 16, {"heuristic": 0}, 7),
    ("uniform", 1500, 24, {"keep_pruned": 0}, 0),
    ("uniform", 1500, 8, {"M": 4}, 64),
    ("grid_ties", 1500, 3, {}, 0),
    ("cosine", 1500, 20, {}, 0),
    ("cosine", 1500, 20, {"heuristic": 0}, 64),
]


def _rows(oracle, kind, n, dim):
    if kind == "grid_ties":
        return datagen.grid_ties(n, dim, 5)
    rows = datagen.uniform(n, dim, 5) - np.float32(0.5)
    return cosine_ref.normalize(oracle, rows) if kind == "cosine" else rows


@pytest.mark.parametrize("kind,n,dim,kw,insert_batch", CONTINUATION)
def test_stopped_build_plus_insert_is_the_full_build(oracle, kind, n, dim, kw, insert_batch):
    rows = _rows(oracle, kind, n, dim)
    mb, gr = S.schedule(insert_batch)
    kw = dict(kw, seed=11)
    full, _ = S.build_batched(rows, mb, gr, threads=4, **kw)
    bounds = layer0_boundaries(oracle, n, kw.get("M", 32), mb, gr)
    picks = sorted({bounds[0], bounds[len(bounds) // 2], bounds[-1]})
    for n0 in picks:
        part, _ = S.build_batched(rows, mb, gr, stop_at=n0, threads=4, **kw)
        assert part.points.shape[0] == n0
        out = S.insert_batched(part, full.points[n0:], mb, gr, threads=4, **kw)
        _same(out, full)


def test_one_insert_per_batch_is_the_sequential_reference_order(oracle):
    rows = datagen.uniform(1200, 12, 9)
    for kw in ({}, {"heuristic": 0}):
        seq, _ = oracle.build(rows, seed=4, **kw)
        g = seq.export()
        n0 = oracle.layer_schedule(1200, 32)[1] + 100
        part, _ = S.build_batched(rows, 1, 8, stop_at=n0, seed=4, **kw)
        _same(S.insert_batched(part, g.points[n0:], 1, 8, **kw), g)


def test_insert_into_an_empty_graph(oracle):
    rows = datagen.uniform(400, 8, 2)
    empty = oracle.Graph(np.zeros((0, 8), np.float32), np.zeros((0, 64), np.uint32), [], 32, 100)
    g = S.insert_batched(empty, rows, 16384, 8)
    assert g.points.tobytes() == rows.tobytes() and g.upper == []
    # the same schedule run as two inserts, split at a batch boundary, gives the same graph (from an empty graph the batches
    # begin at 1, 2, ..., 16, 18, ...)
    g0, b = 1, []
    while g0 < 400:
        b.append(g0)
        g0 += max(1, g0 // 8)
    cut = [x for x in b if x > 100][0]
    two = S.insert_batched(S.insert_batched(empty, rows[:cut], 16384, 8), rows[cut:], 16384, 8)
    _same(two, g)


# ---- recall: what an insert gives up against a full build ----------------------------------------------------------------------
RECALL_N0, RECALL_DIM, RECALL_NQ, RECALL_EF = 4000, 64, 300, 10
# recall@10 (ef_search = 10, where it is well below 1) of n0 built + n0 inserted may trail the full build of the same 2 n0 rows by at
# most this much.  Measured here: full 0.850, inserted 0.870 (the inserted half's rows are re-pruned more often).
RECALL_GAP = 0.02


def recall_case(oracle):
    """(full-build rows in PointId order, n0, queries, ground-truth PointIds) of the recall check; the GPU test reuses it."""
    rows = datagen.sift_shaped(2 * RECALL_N0 + RECALL_NQ, RECALL_DIM, 21, latent=64, noise=0.3)
    pts, q = rows[:2 * RECALL_N0], rows[2 * RECALL_N0:]
    return pts, q


def recall_at_10(ids, truth):
    return float(np.mean([len(set(a[:10].tolist()) & set(b[:10].tolist())) / 10.0 for a, b in zip(ids, truth)]))


def test_insert_recall_stays_within_the_gap_of_a_full_build(oracle):
    pts, q = recall_case(oracle)
    mb, gr = S.schedule(0)
    full, ids = S.build_batched(pts, mb, gr, threads=8, seed=1)
    part, _ = S.build_batched(pts[:RECALL_N0], mb, gr, threads=8, seed=1)
    grown = S.insert_batched(part, pts[RECALL_N0:], mb, gr, threads=8)
    r = {}
    for name, g in (("full", full), ("inserted", grown)):
        truth, _ = oracle.bruteforce(g.points, q, 10, threads=8)
        found = oracle.from_graph(g).search(q, ef_search=RECALL_EF, k=10, threads=8)[0]
        r[name] = recall_at_10(found, truth)
    print(f"recall@10 full {r['full']:.4f}  n0 + n0 inserted {r['inserted']:.4f}")
    assert r["inserted"] >= r["full"] - RECALL_GAP
