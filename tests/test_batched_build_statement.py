"""The CPU statement of the library's batched build schedule (oracle.build_batched, DESIGN.md §6) checked on its own.

tests/test_gpu_batched_build.py compares batched GPU graphs with this statement bit for bit, so the statement is anchored
here: with one insert per batch it must be the sequential oracle build (which the goldens and the reference pins fix), its
graph must not depend on its thread count, its graphs must be well-formed, and its batch boundaries must follow build.cu's
formula.
"""
import numpy as np
import pytest

from tests import datagen

INV = 0xFFFFFFFF


def _same_graph(a, b):
    ga, gb = a.export(), b.export()
    assert ga.points.tobytes() == gb.points.tobytes()
    bad = np.nonzero((ga.zero != gb.zero).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} zero rows differ, first pid {bad[0]}: {ga.zero[bad[0]][:12]} vs {gb.zero[bad[0]][:12]}"
    assert len(ga.upper) == len(gb.upper)
    for x, y in zip(ga.upper, gb.upper):
        assert x.shape == y.shape and (x == y).all()


def _invariants(zero, upper, n, M, layer_counts):
    """The row invariants of tests/test_gpu_build.py, restated so this CPU module does not import a GPU module."""
    assert zero.shape == (n, 2 * M)
    for i, row in enumerate(zero):
        k = int((row != INV).sum())
        assert (row[:k] != INV).all() and (row[k:] == INV).all(), f"row {i} not INVALID-terminated"
        assert len(set(row[:k].tolist())) == k and i not in row[:k] and (row[:k] < n).all()
    assert [n] + [u.shape[0] for u in upper] == layer_counts
    for u in upper:
        assert (u[u != INV] < u.shape[0]).all()


def _schedule(oracle, n, M, max_batch, growth):
    """build.cu's batch loop, restated: per layer top first, b = 1 on the top layer, else min(max_batch, max(1, g0 / growth)),
    clipped to the end of the layer; layer l inserts PointIds [n_{l+1}, n_l), and PointId 0 is never inserted."""
    counts = oracle.layer_schedule(n, M)
    top = len(counts) - 1
    out = []
    for layer in range(top, -1, -1):
        start = max(counts[layer + 1] if layer < top else 0, 1)
        g0 = start
        while g0 < counts[layer]:
            b = 1 if layer == top else min(max_batch, max(1, g0 // growth))
            b = min(b, counts[layer] - g0)
            out.append((g0, b))
            g0 += b
    return out


SEQUENTIAL_CASES = [
    ("uniform", 1500, 16, {}),
    ("uniform", 1500, 16, {"heuristic": 0}),
    ("uniform", 1200, 2, {"heuristic": 0}),
    ("uniform", 1500, 24, {"keep_pruned": 0}),
    ("uniform", 1500, 24, {"ef_construction": 1}),
    ("uniform", 1500, 24, {"ef_construction": 10}),
    ("uniform", 1500, 24, {"ef_construction": 200}),
    ("uniform", 1500, 8, {"M": 8}),
    ("uniform", 2000, 16, {"M": 16}),
    ("uniform", 1500, 32, {"M": 32}),
    ("uniform", 1500, 6, {"M": 64}),
    ("grid_ties", 1500, 3, {}),
    ("grid_ties", 1500, 3, {"heuristic": 0}),
    ("ones", 300, 4, {}),
    ("ones", 300, 4, {"heuristic": 0}),
]


def _data(kind, n, dim, seed):
    if kind == "uniform":
        return datagen.uniform(n, dim, seed)
    if kind == "grid_ties":
        return datagen.grid_ties(n, dim, seed)
    return np.ones((n, dim), dtype=np.float32)


@pytest.mark.parametrize("kind,n,dim,kw", SEQUENTIAL_CASES)
def test_one_insert_per_batch_is_the_sequential_oracle(oracle, kind, n, dim, kw):
    pts = _data(kind, n, dim, 40 + n + dim)
    ix_s, ids_s = oracle.build(pts, seed=n + 1, threads=1, **kw)
    ix_b, ids_b, st = oracle.build_batched(pts, 1, 8, threads=4, seed=n + 1, **kw)
    assert (ids_b == ids_s).all()
    _same_graph(ix_b, ix_s)
    assert st["max_batch"] == 1 and st["batches"] == n - 1
    assert st["multi_new_rounds"] == st["multi_round_targets"] == st["simple_multi_targets"] == 0
    assert st["max_target_requests"] == 1


THREAD_CASES = [
    ("uniform", 6000, 16, {}),
    ("uniform", 6000, 16, {"heuristic": 0}),
    ("uniform", 4000, 24, {"ef_construction": 10}),
    ("grid_ties", 4000, 3, {}),
]


@pytest.mark.parametrize("kind,n,dim,kw", THREAD_CASES)
def test_thread_count_does_not_change_the_batched_graph(oracle, kind, n, dim, kw):
    pts = _data(kind, n, dim, 7)
    ix1, ids1, st1 = oracle.build_batched(pts, 16384, 8, threads=1, seed=3, **kw)
    ix8, ids8, st8 = oracle.build_batched(pts, 16384, 8, threads=8, seed=3, **kw)
    assert (ids1 == ids8).all()
    _same_graph(ix1, ix8)
    for k in st1:
        assert np.array_equal(st1[k], st8[k]), k
    assert st1["max_batch"] > 1


@pytest.mark.parametrize("kind,n,dim,kw,max_batch,growth", [
    ("uniform", 5000, 16, {}, 16384, 8),
    ("uniform", 5000, 16, {"heuristic": 0}, 16384, 8),
    ("uniform", 3000, 8, {"M": 8, "keep_pruned": 0}, 64, 1),
    ("grid_ties", 4000, 3, {}, 16384, 2),
    ("ones", 500, 4, {}, 16384, 8),
])
def test_batched_graphs_are_well_formed(oracle, kind, n, dim, kw, max_batch, growth):
    pts = _data(kind, n, dim, 9)
    ix, ids, st = oracle.build_batched(pts, max_batch, growth, threads=8, seed=5, **kw)
    g = ix.export()
    M = kw.get("M", 32)
    _invariants(g.zero, g.upper, n, M, oracle.layer_schedule(n, M))
    assert sorted(ids.tolist()) == list(range(n))
    # every row was written: by its own insert (PointId 0 is the entry point and is never inserted) or as a target
    assert (st["row_batch"][1:] < st["batches"]).all()


@pytest.mark.parametrize("n,M,max_batch,growth", [
    (1, 32, 16384, 8), (2, 32, 16384, 8), (40, 32, 16384, 8), (5000, 32, 16384, 8), (200_000, 32, 16384, 8),
    (100_000, 24, 16384, 8), (3000, 16, 2, 8), (3000, 16, 7, 8), (3000, 16, 64, 8), (3000, 16, 1000, 8),
    (3000, 16, 16384, 1), (20_000, 8, 100, 3), (5000, 64, 1, 8),
])
def test_batch_boundaries_follow_the_library_formula(oracle, n, M, max_batch, growth):
    pts = datagen.uniform(n, 2, 1)
    _, _, st = oracle.build_batched(pts, max_batch, growth, threads=8, M=M, ef_construction=8)
    want = _schedule(oracle, n, M, max_batch, growth)
    assert [tuple(map(int, b)) for b in st["bounds"]] == want
    assert st["batches"] == len(want) and st["max_batch"] == max((b for _, b in want), default=0)
    assert sum(b for _, b in want) == max(n - 1, 0)


def test_statement_reaches_every_batched_path(oracle):
    """Multi-id rounds, hubs re-pruned in several rounds, admission-limited rounds and simple-mode targets with several requests
    all occur in the statement at the library's default schedule (the GPU module asserts the same on its own cases)."""
    pts = np.repeat(datagen.uniform(4, 8, 2), 2000, axis=0)  # 4 clusters of 2000 exact duplicates
    _, _, st = oracle.build_batched(pts, 16384, 8, threads=8, seed=1, M=8, ef_construction=10)
    assert st["multi_new_rounds"] > 0 and st["multi_round_targets"] > 0 and st["admission_limited_rounds"] > 0
    assert st["max_target_requests"] > 32
    _, _, st = oracle.build_batched(pts, 16384, 8, threads=8, seed=1, M=8, heuristic=0)
    assert st["simple_multi_targets"] > 0 and st["max_target_requests"] > 32


def test_batched_statement_argument_errors(oracle):
    pts = datagen.uniform(100, 4, 1)
    for bad in ({"max_batch": 0, "growth": 8}, {"max_batch": 8, "growth": 0}):
        with pytest.raises(ValueError):
            oracle.build_batched(pts, **bad)
    with pytest.raises(ValueError):
        oracle.build_batched(pts, 8, 8, extend_candidates=1)
    ix, ids, st = oracle.build_batched(np.zeros((0, 4), dtype=np.float32), 8, 8)
    assert ix.n == 0 and len(ids) == 0 and st["batches"] == 0
