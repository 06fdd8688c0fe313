"""q8 row storage (IDB_STORAGE_Q8, DESIGN.md §3c): every row quantised to an 8-bit grid of its own and kept in HBM at a quarter of
the f32 bytes plus an 8-byte header; distances still accumulate in fp32 in the canonical order on the exactly dequantised rows.  Bar:
the device quantiser equals tests/q8_ref.py (pinned on the CPU against an integer-only statement), and everything else is bit for bit
equal to the oracle (and the CPU statements of the batched build, the insert and the sharded merge) run on the DEQUANTISED rows.
Rows with a NaN or infinite element, or whose grid would overflow f32, are refused by the build, the adopt, the insert and the load
with storage q8, before the index changes.

The K1 cells of q8 rows are checked one by one in tests/test_gpu_k1_q8_instantiations.py.
"""
import os

import numpy as np
import pytest

from tests import cosine_ref, datagen, q8_ref
from tests import insert_statement as S
from tests.q8_ref import roundtrip

pytestmark = pytest.mark.gpu
THREADS = min(32, os.cpu_count() or 8)
INVALID = 0xFFFFFFFF
FMAX = np.finfo(np.float32).max


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _flat(abi, pts, storage="q8", metric="l2sq"):
    """An index over `pts` with an empty graph (export and the exact search read the rows only)."""
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    zero = np.full((pts.shape[0], 4), INVALID, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage, metric=metric)


def _schedule(insert_batch):
    if insert_batch:
        return insert_batch, 8
    return (max(1, int(os.environ.get("IDB_BUILD_MAXBATCH", "16384"))), max(1, int(os.environ.get("IDB_BUILD_GROWTH", "8"))))


def _same_graph(ix, g):
    p, zero, upper = ix.export_graph()
    assert p.shape == g.points.shape and p.tobytes() == g.points.tobytes(), "stored rows differ"
    bad = np.nonzero((zero != g.zero).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} zero rows differ, first PointId {bad[0]}"
    assert len(upper) == len(g.upper) and all(a.shape == b.shape and (a == b).all() for a, b in zip(upper, g.upper))


def _same_search(got, want):
    ids, dist, lens = got[:3]
    assert (lens == want[2]).all() and (ids == want[0]).all() and dist.tobytes() == want[1].tobytes()


def _same_exact(got, want_ids, want_dist):
    ids, dist, lens = got
    assert (ids == want_ids).all() and dist.tobytes() == np.ascontiguousarray(want_dist, np.float32).tobytes()
    assert (lens == (want_ids != INVALID).sum(1)).all()


def _same_rows(got, want):
    g, w = got.view(np.uint32).ravel(), np.ascontiguousarray(want, np.float32).view(np.uint32).ravel()
    bad = np.nonzero(g != w)[0]
    assert len(bad) == 0, f"{len(bad)} elements differ; first (index, q8_ref, stored) bits: " + ", ".join(
        f"({i}, {w[i]:#x}, {g[i]:#x})" for i in bad[:6])


def _mixed_rows(n, dim, seed):
    """n rows of mixed kinds and scales (2^-140 .. 2^100), subnormal and constant rows included."""
    r = np.random.default_rng(seed)
    kind = np.arange(n) % 5
    scale = np.ldexp(np.float32(1), r.integers(-140, 100, n)).astype(np.float32)[:, None]
    x = r.standard_normal((n, dim)).astype(np.float32) * scale
    x[kind == 1] = np.abs(x[kind == 1])
    x[kind == 2] = np.float32(1000) + r.standard_normal(((kind == 2).sum(), dim)).astype(np.float32) * np.float32(1e-3)
    x[kind == 3] = x[kind == 3][:, :1]
    tiny = kind == 4
    x[tiny] = r.standard_normal((tiny.sum(), dim)).astype(np.float32) * np.ldexp(np.float32(1), r.integers(-149, -125, (tiny.sum(), dim)))
    return x.astype(np.float32)


# ---- 1. the quantiser ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [1, 3, 8, 37, 128])
def test_quantiser_equals_q8_ref_on_the_boundary_set(abi, dim):
    x = q8_ref.boundary_rows(dim)
    accepted = q8_ref.overflow_rows(max(dim, 2))[1][:, :dim]
    x = np.concatenate([x, accepted, _mixed_rows(200, dim, dim)])
    ix = _flat(abi, x)
    assert ix.info().storage == abi.STORAGE["q8"]
    _same_rows(ix.export_graph()[0], roundtrip(x))
    # idempotent: the dequantised rows, quantised again, are the same rows
    again = _flat(abi, ix.export_graph()[0])
    _same_rows(again.export_graph()[0], roundtrip(x))


def test_quantiser_equals_q8_ref_on_a_million_rows(abi):
    x = _mixed_rows(1_000_000, 16, 3)
    ix = _flat(abi, x)
    _same_rows(ix.export_graph()[0], roundtrip(x))


# ---- 2. refusals -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bad", ["nan", "inf", "-inf", "fmax"])
def test_refused_rows_by_build_adopt_insert_and_load(abi, bad, tmp_path):
    rows = datagen.uniform(300, 20, 3)
    poisoned = rows.copy()
    poisoned[123, 7] = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf, "fmax": FMAX}[bad]
    assert q8_ref.refused(poisoned[123:124]).all()
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(poisoned, storage="q8", seed=1)
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    zero = np.full((300, 64), INVALID, np.uint32)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(poisoned, zero, [], 32, storage="q8")
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    # the insert refuses the rows and leaves n, the rows, the graph and the search as they were
    ix, _ = abi.Index.build(rows[:200], storage="q8", seed=1)
    q = datagen.uniform(20, 20, 4)
    before = ix.export_graph(), ix.search(q, ef_search=50, k=10)
    for n in (200, 210):  # the second time after an insert that grew the storage
        with pytest.raises(abi.IdbError) as e:
            ix.insert(poisoned[100:200])
        assert e.value.status == abi.ERR_INVALID_ARG and "row 23, element 7" in str(e.value)
        after = ix.export_graph(), ix.search(q, ef_search=50, k=10)
        assert int(ix.info().n) == n
        assert after[0][0].tobytes() == before[0][0].tobytes() and (after[0][1] == before[0][1]).all()
        assert all((a == b).all() for a, b in zip(after[0][2], before[0][2]))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(after[1], before[1]))
        ix.insert(rows[200:210])
        before = ix.export_graph(), ix.search(q, ef_search=50, k=10)
    if bad == "fmax":  # a finite file: loads as f32, refused as q8
        path = str(tmp_path / "big.idx")
        _flat(abi, poisoned, storage="f32").save(path)
        with pytest.raises(abi.IdbError) as e:
            abi.Index.load(path, dim=20, M=2, storage="q8")
        assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
        abi.Index.load(path, dim=20, M=2)[0].close()


def test_overflow_threshold_on_the_device(abi):
    refused, accepted = q8_ref.overflow_rows()
    for i, row in enumerate(refused):
        with pytest.raises(abi.IdbError) as e:
            _flat(abi, np.concatenate([accepted, row[None, :]]))
        assert e.value.status == abi.ERR_INVALID_ARG and f"row {len(accepted)}," in str(e.value), i
    ix = _flat(abi, accepted)
    _same_rows(ix.export_graph()[0], roundtrip(accepted))


# ---- 3. build ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,dim", [(1500, 128), (1000, 77), (500, 1536)])
def test_sequential_build_equals_the_oracle_on_dequantised_rows(abi, oracle, n, dim):
    pts = datagen.uniform(n, dim, 8) * np.float32(3.7)
    ix_o, ids_o = oracle.build(roundtrip(pts), seed=12, threads=1)
    g = ix_o.export()
    ix, ids = abi.Index.build(pts, seed=12, insert_batch=1, storage="q8")
    p, zero, upper = ix.export_graph()
    assert (ids == ids_o).all() and p.tobytes() == g.points.tobytes() and (zero == g.zero).all()
    assert all((a == b).all() for a, b in zip(upper, g.upper))


@pytest.mark.parametrize("case", ["default", "insert_batch 64", "simple", "keep_pruned 0", "cosine", "dim 45"])
def test_batched_build_equals_the_statement_on_dequantised_rows(abi, oracle, case):
    dim = 64 if case == "cosine" else 45 if case == "dim 45" else 128
    rows = datagen.sift_shaped(5000 if case != "cosine" else 4000, dim, 800)
    kw, metric, insert_batch = {"seed": 10}, "l2sq", 0
    if case == "insert_batch 64":
        insert_batch = 64
    if case == "simple":
        kw["heuristic"] = 0
    if case == "keep_pruned 0":
        kw["keep_pruned"] = 0
    if case == "cosine":
        metric = "cosine"
    stored = cosine_ref.normalize(oracle, rows) if metric == "cosine" else rows  # normalised in f32, then quantised
    mb, gr = _schedule(insert_batch)
    ix_o, ids_o, st = oracle.build_batched(roundtrip(stored), mb, gr, threads=THREADS, **kw)
    ix, ids = abi.Index.build(rows, insert_batch=insert_batch, metric=metric, storage="q8", **kw)
    assert (ids == ids_o).all()
    _same_graph(ix, ix_o.export())
    assert st["max_batch"] > 1


# ---- 4. insert ---------------------------------------------------------------------------------------------------------------

def test_insert_continuation_equals_the_statement(abi, oracle):
    from tests.test_insert_statement import layer0_boundaries

    rows = datagen.sift_shaped(4000, 128, 168)
    mb, gr = _schedule(0)
    stored = roundtrip(rows)
    full, ids = S.build_batched(stored, mb, gr, threads=THREADS, seed=3)
    bounds = layer0_boundaries(oracle, 4000, 32, mb, gr)
    n0 = bounds[len(bounds) // 2]
    part, _ = S.build_batched(stored, mb, gr, stop_at=n0, threads=THREADS, seed=3)
    ix = abi.Index.from_graph(part.points, part.zero, part.upper, part.M, ef_search=part.ef_search, storage="q8")
    assert (ix.insert(rows[np.argsort(ids)][n0:]) == np.arange(n0, 4000)).all()
    _same_graph(ix, full)


def test_empty_q8_index_stays_q8_across_successive_inserts(abi, oracle):
    rows = datagen.uniform(5000, 23, 8) * np.float32(3.3)
    ix, _ = abi.Index.build(np.zeros((0, 23), np.float32), storage="q8")
    assert ix.info().storage == abi.STORAGE["q8"]
    g = oracle.Graph(np.zeros((0, 23), np.float32), np.zeros((0, 64), np.uint32), [], 32, 100)
    mb, gr = _schedule(0)
    for a, b in ((0, 1), (1, 2), (2, 40), (40, 41), (41, 700), (700, 5000)):  # across several capacity doublings
        assert (ix.insert(rows[a:b]) == np.arange(a, b)).all()
        g = S.insert_batched(g, roundtrip(rows[a:b]), mb, gr, threads=THREADS)
        _same_graph(ix, g)
    assert ix.info().storage == abi.STORAGE["q8"]


# ---- 5. exact search ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [3, 128, 129, 300, 640, 768, 1024, 1025, 4100])
def test_exact_search_every_kernel_cell(abi, oracle, dim):
    pts = datagen.uniform(2500, dim, 1) * np.float32(5.1) - np.float32(1.3)
    q = datagen.uniform(37, dim, 2) * np.float32(5.1)
    ix = _flat(abi, pts)
    _same_exact(ix.exact_search(q, 10), *oracle.bruteforce(roundtrip(pts), q, 10, threads=THREADS))


# ---- 6. sharded: f32, bf16, fp16 and q8 shards in one call -----------------------------------------------------------------

def test_sharded_mixed_row_types(abi, oracle):
    """The fused path against the plain merge of the oracle's per-shard lists (tests/merge_statement.py), each shard searched by the
    oracle on its own stored rows, with the K1 cell of its row type (tests/k1_dispatch_q8.py) and the oracle's per-layer counters."""
    from tests import merge_statement as ms
    from tests.k1_dispatch import Cell
    from tests.k1_dispatch_q8 import k1_cell
    from tests.test_gpu_sharded import Spec, _oracle_keys, _queries, _shards

    comm = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    specs = [Spec(1200, 100), Spec(1100, 100, "bf16"), Spec(1000, 100, "f16"), Spec(900, 100, "q8", M=32), Spec(800, 100, "q8")]
    shards = _shards(abi, oracle, specs)
    try:
        for sh in shards[3:]:
            assert sh.ix.info().storage == abi.STORAGE["q8"]
        ef, k = 64, 20
        for kind in ("sift", "rows"):
            q = _queries(shards, 64, kind, 77)
            got = abi.sharded_search_multi([sh.ix for sh in shards], comm, q, ef_search=ef, k=k)
            keys = []
            for i, sh in enumerate(shards):
                kk, cnt = _oracle_keys(oracle, sh, q, ef, k)
                keys.append(kk)
                assert Cell(**sh.ix.last_kernel()) == k1_cell(sh.spec.dim, sh.spec.M, ef, sh.spec.n, sh.spec.storage), f"shard {i}"
                assert (sh.ix.last_counters(len(q)) == cnt).all(), f"shard {i}: per-layer counters differ"
            _same_search(got, ms.merge(np.stack(keys), k, "l2sq"))
    finally:
        for sh in shards:
            sh.ix.close()
        comm.close()


# ---- 7. save / load ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", ["l2sq", "cosine"])
def test_save_load_and_save_again(abi, oracle, tmp_path, metric):
    rows = datagen.sift_shaped(3000, 128, 21)
    q = datagen.sift_shaped(100, 128, 22)
    ix, _ = abi.Index.build(rows, storage="q8", seed=4, metric=metric)
    path = str(tmp_path / "q8.idx")
    ix.save(path)
    ld, off = abi.Index.load(path, dim=128, M=32, storage="q8", metric=metric)
    assert ld.info().storage == abi.STORAGE["q8"] and off == os.path.getsize(path)
    a, b = ix.export_graph(), ld.export_graph()
    assert a[0].tobytes() == b[0].tobytes() and (a[1] == b[1]).all() and all((x == y).all() for x, y in zip(a[2], b[2]))
    _same_search(ld.search(q, ef_search=100, k=10), ix.search(q, ef_search=100, k=10))
    _same_search(ld.exact_search(q, 10), ix.exact_search(q, 10))
    ld.save(str(tmp_path / "again.idx"))
    assert open(path, "rb").read() == open(str(tmp_path / "again.idx"), "rb").read()
    # the file holds the dequantised rows: loaded as f32 they are the same values
    f32, _ = abi.Index.load(path, dim=128, M=32, metric=metric)
    assert f32.info().storage == abi.STORAGE["f32"] and f32.export_graph()[0].tobytes() == a[0].tobytes()


# ---- 8. no screening table ---------------------------------------------------------------------------------------------------

def test_no_screening_table_every_candidate_fetched_in_full(abi, oracle):
    rows = datagen.sift_shaped(4000, 128, 61)
    q = datagen.sift_shaped(200, 128, 62)
    ix, _ = abi.Index.build(rows, storage="q8", seed=5)
    p, zero, upper = ix.export_graph()
    ox = oracle.from_graph(oracle.Graph(p, zero, upper, 32, 100))
    _same_search(ix.search(q, ef_search=100, k=10), ox.search(q, ef_search=100, k=10, threads=THREADS))
    cnt = ix.last_counters(len(q))
    assert ix.last_full_fetches() == int(cnt[:, 1].sum() + cnt[:, 3].sum())
    with pytest.raises(abi.IdbError) as e:
        ix.screen_bound(q[:1], np.uint32([[0, 0]]))
    assert e.value.status == abi.ERR_UNSUPPORTED


# ---- 9. the Python module ------------------------------------------------------------------------------------------------

def test_python_module_with_q8_storage(abi, oracle, tmp_path):
    import instant_distance as idist

    rows = datagen.sift_shaped(2000, 64, 31)
    cfg = idist.Config()
    cfg.storage, cfg.seed = "q8", 9
    h, ids = idist.Hnsw.build(rows[:1500].tolist(), cfg)
    assert h._ix.info().storage == abi.STORAGE["q8"]
    ids_o = np.asarray(ids)
    g = h._ix.export_graph()
    assert g[0].tobytes() == roundtrip(rows[:1500])[np.argsort(ids_o)].tobytes()
    q = datagen.sift_shaped(30, 64, 32)
    ox = oracle.from_graph(oracle.Graph(g[0], g[1], g[2], 32, 100))
    _same_search(h.search_many(q, k=10), ox.search(q, ef_search=100, k=10, threads=THREADS))
    _same_exact(h.search_exact(q, k=10), *oracle.bruteforce(g[0], q, 10))
    assert h.insert(rows[1500:].tolist()) == list(range(1500, 2000))
    path = str(tmp_path / "m.idx")
    h.dump(path)
    ld = idist.Hnsw.load(path, dim=64, M=32, storage="q8")
    assert ld._ix.info().storage == abi.STORAGE["q8"]
    assert ld._ix.export_graph()[0].tobytes() == h._ix.export_graph()[0].tobytes()
    _same_search(ld.search_many(q, k=10), h.search_many(q, k=10))
    hm = idist.HnswMap.build(rows[:500].tolist(), [str(i) for i in range(500)], cfg)
    hm.dump(path)
    lm = idist.HnswMap.load(path, dim=64, M=32, storage="q8")
    assert lm.values == hm.values and lm._ix.info().storage == abi.STORAGE["q8"]
