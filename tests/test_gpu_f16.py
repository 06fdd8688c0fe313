"""fp16 row storage (IDB_STORAGE_F16, DESIGN.md §3b): rows rounded to fp16 (RNE, subnormals kept) and kept in HBM at half the bytes;
distances still accumulate in fp32 in the canonical order on the exactly widened rows.  Bar: bit for bit equal to the oracle (and
the CPU statements of the batched build, the insert and the sharded merge) run on the fp16-ROUNDED rows, which numpy's
`astype(np.float16)` gives (tests/test_f16_cpu.py pins it against an integer statement of the rounding).  Values that would round
to infinity are refused by the build, the adopt, the insert and the load with storage f16, before the index changes.

The K1 cells of fp16 rows are checked one by one in tests/test_gpu_k1_f16_instantiations.py.
"""
import os

import numpy as np
import pytest

from tests import cosine_ref, datagen, f16_ref
from tests import insert_statement as S
from tests.f16_ref import f16_round

pytestmark = pytest.mark.gpu
THREADS = min(32, os.cpu_count() or 8)
INVALID = 0xFFFFFFFF


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _flat(abi, pts, storage="f16", metric="l2sq"):
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


# ---- 1. narrowing ---------------------------------------------------------------------------------------------------------

def test_narrowing_equals_numpy_on_the_boundary_set(abi):
    x = f16_ref.boundary_values()
    x = np.concatenate([x, np.float32([np.inf, -np.inf, np.nan, -np.nan, 0.0, -0.0])])
    x = np.concatenate([x, np.zeros((-len(x)) % 128, np.float32)]).reshape(-1, 128)
    ix = _flat(abi, x)
    assert ix.info().storage == abi.STORAGE["f16"]
    got, want = ix.export_graph()[0].view(np.uint32).ravel(), f16_round(x).view(np.uint32).ravel()
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, (f"{len(bad)} elements differ; first (input, numpy, stored) bits: " +
                           ", ".join(f"({x.view(np.uint32).ravel()[i]:#x}, {want[i]:#x}, {got[i]:#x})" for i in bad[:6]))
    got = got.view(np.float32).reshape(x.shape)
    flat = x.ravel()
    assert got.ravel()[flat == np.nextafter(np.float32(65520), np.float32(0))].tolist() == [65504.0]


@pytest.mark.parametrize("bad", [65520.0, -70000.0])
def test_values_beyond_fp16_are_refused_by_build_adopt_and_insert(abi, bad):
    rows = datagen.uniform(300, 20, 3)
    poisoned = rows.copy()
    poisoned[123, 7] = bad
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(poisoned, storage="f16", seed=1)
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    zero = np.full((300, 64), INVALID, np.uint32)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(poisoned, zero, [], 32, storage="f16")
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    # the insert refuses the rows and leaves n, the rows, the graph and the search as they were
    ix, _ = abi.Index.build(rows[:200], storage="f16", seed=1)
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
    # bf16 and f32 take the same rows
    for storage in ("f32", "bf16"):
        abi.Index.build(poisoned, storage=storage, seed=1)[0].close()


# ---- 2. widening in the kernels: every finite fp16 value ------------------------------------------------------------------

def test_every_finite_fp16_value_through_k1_and_the_exact_search(abi, oracle):
    h = np.arange(0x10000, dtype=np.uint32).astype(np.uint16)
    v = h.view(np.float16)
    vals = v[np.isfinite(v)].astype(np.float32)  # 63 488 values, +-0 and the subnormals included
    assert len(vals) == 63488
    vals = vals[np.random.default_rng(5).permutation(len(vals))]
    pts = vals.reshape(-1, 128)  # 496 rows
    ix, _ = abi.Index.build(pts, storage="f16", seed=3, M=16)
    p, zero, upper = ix.export_graph()
    assert p.tobytes() != pts.tobytes() and (np.sort(p.view(np.uint32).ravel()) == np.sort(pts.view(np.uint32).ravel())).all()
    ox = oracle.from_graph(oracle.Graph(p, zero, upper, 16, 100))
    q = np.concatenate([p[::9] * np.float32(0.5), datagen.uniform(20, 128, 6) * np.float32(1000)]).astype(np.float32)
    _same_search(ix.search(q, ef_search=64, k=64), ox.search(q, ef_search=64, k=64, threads=THREADS))
    _same_exact(ix.exact_search(q, 50), *oracle.bruteforce(p, q, 50, threads=THREADS))
    # the small values alone: subnormal rows against subnormal-scale queries
    small = np.sort(np.abs(vals))[:128 * 8].reshape(8, 128)
    fx = _flat(abi, small)
    assert fx.export_graph()[0].tobytes() == small.tobytes()
    qs = small[::-1] * np.float32(0.75)
    _same_exact(fx.exact_search(qs, 8), *oracle.bruteforce(small, qs, 8))


# ---- 4. build ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,dim", [(1500, 128), (1000, 768), (500, 1536)])
def test_sequential_build_equals_the_oracle_on_rounded_rows(abi, oracle, n, dim):
    pts = datagen.uniform(n, dim, 8) * np.float32(3.7)
    ix_o, ids_o = oracle.build(f16_round(pts), seed=12, threads=1)
    g = ix_o.export()
    ix, ids = abi.Index.build(pts, seed=12, insert_batch=1, storage="f16")
    p, zero, upper = ix.export_graph()
    assert (ids == ids_o).all() and p.tobytes() == g.points.tobytes() and (zero == g.zero).all()
    assert all((a == b).all() for a, b in zip(upper, g.upper))


@pytest.mark.parametrize("case", ["default", "insert_batch 64", "simple", "keep_pruned 0", "cosine"])
def test_batched_build_equals_the_statement_on_rounded_rows(abi, oracle, case):
    rows = datagen.sift_shaped(5000, 128, 800) if case != "cosine" else datagen.sift_shaped(4000, 64, 900)
    kw, metric, insert_batch = {"seed": 10}, "l2sq", 0
    if case == "insert_batch 64":
        insert_batch = 64
    if case == "simple":
        kw["heuristic"] = 0
    if case == "keep_pruned 0":
        kw["keep_pruned"] = 0
    if case == "cosine":
        metric = "cosine"
    stored = cosine_ref.normalize(oracle, rows) if metric == "cosine" else rows  # normalised in f32, then rounded
    mb, gr = _schedule(insert_batch)
    ix_o, ids_o, st = oracle.build_batched(f16_round(stored), mb, gr, threads=THREADS, **kw)
    ix, ids = abi.Index.build(rows, insert_batch=insert_batch, metric=metric, storage="f16", **kw)
    assert (ids == ids_o).all()
    _same_graph(ix, ix_o.export())
    assert st["max_batch"] > 1


# ---- 5. insert ---------------------------------------------------------------------------------------------------------------

def test_insert_continuation_equals_the_statement(abi, oracle):
    from tests.test_insert_statement import layer0_boundaries

    rows = datagen.sift_shaped(4000, 128, 168)
    mb, gr = _schedule(0)
    stored = f16_round(rows)
    full, ids = S.build_batched(stored, mb, gr, threads=THREADS, seed=3)
    bounds = layer0_boundaries(oracle, 4000, 32, mb, gr)
    n0 = bounds[len(bounds) // 2]
    part, _ = S.build_batched(stored, mb, gr, stop_at=n0, threads=THREADS, seed=3)
    ix = abi.Index.from_graph(part.points, part.zero, part.upper, part.M, ef_search=part.ef_search, storage="f16")
    assert (ix.insert(rows[np.argsort(ids)][n0:]) == np.arange(n0, 4000)).all()
    _same_graph(ix, full)


def test_empty_f16_index_stays_f16_across_successive_inserts(abi, oracle):
    rows = datagen.uniform(5000, 24, 8) * np.float32(3.3)
    ix, _ = abi.Index.build(np.zeros((0, 24), np.float32), storage="f16")
    assert ix.info().storage == abi.STORAGE["f16"]
    g = oracle.Graph(np.zeros((0, 24), np.float32), np.zeros((0, 64), np.uint32), [], 32, 100)
    mb, gr = _schedule(0)
    for a, b in ((0, 1), (1, 2), (2, 40), (40, 41), (41, 700), (700, 5000)):  # across several capacity doublings
        assert (ix.insert(rows[a:b]) == np.arange(a, b)).all()
        g = S.insert_batched(g, f16_round(rows[a:b]), mb, gr, threads=THREADS)
        _same_graph(ix, g)
    assert ix.info().storage == abi.STORAGE["f16"]


# ---- 6. exact search ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [3, 128, 129, 300, 640, 768, 1024, 1025, 4100])
def test_exact_search_every_kernel_cell(abi, oracle, dim):
    pts = datagen.uniform(2500, dim, 1) * np.float32(5.1)
    q = datagen.uniform(37, dim, 2) * np.float32(5.1)
    ix = _flat(abi, pts)
    _same_exact(ix.exact_search(q, 10), *oracle.bruteforce(f16_round(pts), q, 10, threads=THREADS))


# ---- 7. sharded: f32, bf16 and fp16 shards in one call ------------------------------------------------------------------

def test_sharded_mixed_row_types(abi, oracle):
    """The fused path against the plain merge of the oracle's per-shard lists (tests/merge_statement.py), each shard searched by the
    oracle on its own stored rows, with the K1 cell of its row type (tests/k1_dispatch_f16.py) and the oracle's per-layer counters."""
    from tests import merge_statement as ms
    from tests.k1_dispatch import Cell
    from tests.k1_dispatch_f16 import k1_cell
    from tests.test_gpu_sharded import Spec, _oracle_keys, _queries, _shards

    comm = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    specs = [Spec(1200, 100), Spec(1100, 100, "bf16"), Spec(1000, 100, "f16"), Spec(900, 100, "f16", M=32)]
    shards = _shards(abi, oracle, specs)
    try:
        for sh in shards[2:]:
            assert sh.ix.info().storage == abi.STORAGE["f16"]
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


# ---- 8. save / load ----------------------------------------------------------------------------------------------------------

def test_save_and_load_with_the_storage(abi, oracle, tmp_path):
    rows = datagen.sift_shaped(3000, 128, 21)
    q = datagen.sift_shaped(100, 128, 22)
    for storage in ("f16", "bf16"):
        ix, _ = abi.Index.build(rows, storage=storage, seed=4)
        path = str(tmp_path / f"{storage}.idx")
        ix.save(path)
        ld, off = abi.Index.load(path, dim=128, M=32, storage=storage)
        assert ld.info().storage == abi.STORAGE[storage] and off == os.path.getsize(path)
        a, b = ix.export_graph(), ld.export_graph()
        assert a[0].tobytes() == b[0].tobytes() and (a[1] == b[1]).all() and all((x == y).all() for x, y in zip(a[2], b[2]))
        _same_search(ld.search(q, ef_search=100, k=10), ix.search(q, ef_search=100, k=10))
        _same_search(ld.exact_search(q, 10), ix.exact_search(q, 10))
        # load_ex (and load with the default storage) still gives f32 rows, holding the same values
        f32, _ = abi.Index.load(path, dim=128, M=32)
        assert f32.info().storage == abi.STORAGE["f32"] and f32.export_graph()[0].tobytes() == a[0].tobytes()
        ld.save(str(tmp_path / "again.idx"))
        assert open(path, "rb").read() == open(str(tmp_path / "again.idx"), "rb").read()
    # a file with values beyond fp16 loads as f32 and bf16 and is refused as f16
    big = rows * np.float32(10000)
    ix, _ = abi.Index.build(big, seed=4)
    path = str(tmp_path / "big.idx")
    ix.save(path)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.load(path, dim=128, M=32, storage="f16")
    assert e.value.status == abi.ERR_INVALID_ARG
    abi.Index.load(path, dim=128, M=32, storage="bf16")[0].close()


# ---- 9. the Python module ------------------------------------------------------------------------------------------------

def test_python_module_with_f16_storage(abi, oracle, tmp_path):
    import instant_distance as idist

    rows = datagen.sift_shaped(2000, 64, 31)
    cfg = idist.Config()
    cfg.storage, cfg.seed = "f16", 9
    h, ids = idist.Hnsw.build(rows[:1500].tolist(), cfg)
    assert h._ix.info().storage == abi.STORAGE["f16"]
    ids_o = np.asarray(ids)
    g = h._ix.export_graph()
    assert g[0].tobytes() == f16_round(rows[:1500])[np.argsort(ids_o)].tobytes()
    q = datagen.sift_shaped(30, 64, 32)
    ox = oracle.from_graph(oracle.Graph(g[0], g[1], g[2], 32, 100))
    _same_search(h.search_many(q, k=10), ox.search(q, ef_search=100, k=10, threads=THREADS))
    _same_exact(h.search_exact(q, k=10), *oracle.bruteforce(g[0], q, 10))
    assert h.insert(rows[1500:].tolist()) == list(range(1500, 2000))
    path = str(tmp_path / "m.idx")
    h.dump(path)
    ld = idist.Hnsw.load(path, dim=64, M=32, storage="f16")
    assert ld._ix.info().storage == abi.STORAGE["f16"]
    assert ld._ix.export_graph()[0].tobytes() == h._ix.export_graph()[0].tobytes()
    _same_search(ld.search_many(q, k=10), h.search_many(q, k=10))
    s = idist.Search()
    ld.search(q[0].tolist(), s)
    assert [n.pid for n in s][:10] == h.search_many(q[:1], k=10)[0][0].tolist()
    hm = idist.HnswMap.build(rows[:500].tolist(), [str(i) for i in range(500)], cfg)
    hm.dump(path)
    lm = idist.HnswMap.load(path, dim=64, M=32, storage="f16")
    assert lm.values == hm.values and lm._ix.info().storage == abi.STORAGE["f16"]


# ---- 10. recall: fp16 against bf16, both against the f32 exact search --------------------------------------------------

def test_f16_recall_is_not_below_bf16(abi):
    rows = datagen.sift_shaped(20000, 128, 3)
    q = datagen.sift_shaped(300, 128, 4)
    ix32, ids32 = abi.Index.build(rows, seed=2)
    truth = ix32.exact_search(q, 10)[0]  # PointIds of the f32 index; the same seed gives every storage the same PointIds
    rec = {}
    for storage in ("bf16", "f16"):
        ix, ids = abi.Index.build(rows, seed=2, storage=storage)
        assert (ids == ids32).all()
        got = ix.search(q, ef_search=100, k=10)[0]
        rec[storage] = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(got, truth)]))
    print(f"recall@10 against the f32 exact search: bf16 {rec['bf16']:.4f}, f16 {rec['f16']:.4f}")
    assert rec["f16"] >= rec["bf16"] - 0.002, rec
