"""bin row storage (IDB_STORAGE_BIN, DESIGN.md §3d): 0/1 rows kept at one byte per four elements.  The statement throughout is the
existing f32 oracle (and the CPU statements of the batched build, the insert, the removal, the range search and the sharded merge) on
the same 0/1 rows, bit for bit; for 0/1 queries the reported distances are also checked against numpy popcount Hamming distances.
Values other than +-0 and 1 are refused by the build, the adopt, the insert and the load, before the index changes; cosine with bin
is refused.  Heavy exact ties (dims 4, 16, 37, duplicate rows) reach the tie lists and the retry pass.

The K1 cells of bin rows are checked one by one in tests/test_gpu_k1_bin_instantiations.py.
"""
import os

import numpy as np
import pytest

from tests import bin_ref, datagen, range_ref
from tests import insert_statement as S
from tests import remove_ref as R

pytestmark = pytest.mark.gpu
THREADS = min(32, os.cpu_count() or 8)
INVALID = 0xFFFFFFFF


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _bits(n, dim, seed, q=0):
    """n sift-shaped rows binarised at their column medians (q > 0: also q queries binarised at the same medians)."""
    raw = datagen.sift_shaped(n + q, dim, seed)
    x = bin_ref.binarise(raw, raw[:n])
    return (x[:n], x[n:]) if q else x


def _flat(abi, pts, storage="bin"):
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    zero = np.full((pts.shape[0], 4), INVALID, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage)


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


def _oracle(oracle, ix, M=32):
    p, zero, upper = ix.export_graph()
    return oracle.from_graph(oracle.Graph(p, zero, upper, M, 100))


# ---- 1. rows in and out ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [1, 3, 4, 16, 37, 128, 300, 1025])
def test_export_returns_the_0_1_rows(abi, dim):
    x = (np.random.default_rng(dim).random((700, dim)) < 0.5).astype(np.float32)
    x[0] = 1.0
    x[1] = -0.0  # stored as +0
    ix = _flat(abi, x)
    assert ix.info().storage == abi.STORAGE["bin"] == 8
    got = ix.export_graph()[0]
    assert got.tobytes() == (x + np.float32(0)).tobytes()  # -0 + 0 = +0
    assert got.tobytes() == bin_ref.unpack(bin_ref.pack(x), dim).tobytes()


# ---- 2. refusals -------------------------------------------------------------------------------------------------------------

BAD = {"0.5": 0.5, "2": 2.0, "-1": -1.0, "nan": np.nan, "inf": np.inf, "-inf": -np.inf,
       "subnormal": float(np.finfo(np.float32).smallest_subnormal), "next1": float(np.nextafter(np.float32(1), np.float32(2)))}


@pytest.mark.parametrize("bad", list(BAD))
def test_refused_rows_by_build_adopt_insert_and_load(abi, bad, tmp_path):
    rows = _bits(300, 20, 3)
    poisoned = rows.copy()
    poisoned[123, 7] = BAD[bad]
    assert bin_ref.refused(poisoned[123:124]).sum() == 1
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(poisoned, storage="bin", seed=1)
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    zero = np.full((300, 64), INVALID, np.uint32)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(poisoned, zero, [], 32, storage="bin")
    assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
    # the insert refuses the rows and leaves n, the rows, the graph, the id map and the search as they were
    ix, _ = abi.Index.build(rows[:200], storage="bin", seed=1)
    ix.set_id_map(np.arange(1000, 1200, dtype=np.uint32))
    q = _bits(20, 20, 4)
    before = ix.export_graph(), ix.search(q, ef_search=50, k=10)
    for n in (200, 210):  # the second time after an insert that grew the storage
        with pytest.raises(abi.IdbError) as e:
            ix.insert(poisoned[100:200], global_ids=np.arange(5000, 5100, dtype=np.uint32))
        assert e.value.status == abi.ERR_INVALID_ARG and "row 23, element 7" in str(e.value)
        after = ix.export_graph(), ix.search(q, ef_search=50, k=10)
        assert int(ix.info().n) == n
        assert after[0][0].tobytes() == before[0][0].tobytes() and (after[0][1] == before[0][1]).all()
        assert all((a == b).all() for a, b in zip(after[0][2], before[0][2]))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(after[1], before[1]))  # ids come through the id map
        ix.insert(rows[200:210], global_ids=np.arange(1200, 1210, dtype=np.uint32))
        before = ix.export_graph(), ix.search(q, ef_search=50, k=10)
    if np.isfinite(BAD[bad]):  # a file of finite rows: loads as f32, refused as bin
        path = str(tmp_path / "bad.idx")
        _flat(abi, poisoned, storage="f32").save(path)
        with pytest.raises(abi.IdbError) as e:
            abi.Index.load(path, dim=20, M=2, storage="bin")
        assert e.value.status == abi.ERR_INVALID_ARG and "row 123, element 7" in str(e.value)
        abi.Index.load(path, dim=20, M=2)[0].close()


def test_cosine_with_bin_is_refused(abi, tmp_path):
    rows = _bits(100, 16, 5)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(rows, storage="bin", metric="cosine")
    assert e.value.status == abi.ERR_UNSUPPORTED
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(rows, np.full((100, 4), INVALID, np.uint32), [], 2, storage="bin", metric="cosine")
    assert e.value.status == abi.ERR_UNSUPPORTED
    path = str(tmp_path / "c.idx")
    _flat(abi, rows).save(path)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.load(path, dim=16, M=2, storage="bin", metric="cosine")
    assert e.value.status == abi.ERR_UNSUPPORTED


# ---- 3. build ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,dim", [(1500, 128), (1000, 37), (500, 1536)])
def test_sequential_build_equals_the_oracle(abi, oracle, n, dim):
    pts = _bits(n, dim, 8)
    ix_o, ids_o = oracle.build(pts, seed=12, threads=1)
    g = ix_o.export()
    ix, ids = abi.Index.build(pts, seed=12, insert_batch=1, storage="bin")
    assert (ids == ids_o).all()
    _same_graph(ix, g)


@pytest.mark.parametrize("case", ["default", "insert_batch 64", "simple", "keep_pruned 0", "dim 16", "dim 4"])
def test_batched_build_equals_the_statement(abi, oracle, case):
    dim = {"dim 16": 16, "dim 4": 4}.get(case, 128)
    rows = _bits(5000, dim, 800)
    kw, insert_batch = {"seed": 10}, 0
    if case == "insert_batch 64":
        insert_batch = 64
    if case == "simple":
        kw["heuristic"] = 0
    if case == "keep_pruned 0":
        kw["keep_pruned"] = 0
    mb, gr = _schedule(insert_batch)
    ix_o, ids_o, st = oracle.build_batched(rows, mb, gr, threads=THREADS, **kw)
    ix, ids = abi.Index.build(rows, insert_batch=insert_batch, storage="bin", **kw)
    assert (ids == ids_o).all()
    _same_graph(ix, ix_o.export())
    assert st["max_batch"] > 1


# ---- 4. insert and remove ----------------------------------------------------------------------------------------------------

def test_insert_continuation_equals_the_statement(abi, oracle):
    from tests.test_insert_statement import layer0_boundaries

    rows = _bits(4000, 128, 168)
    mb, gr = _schedule(0)
    full, ids = S.build_batched(rows, mb, gr, threads=THREADS, seed=3)
    bounds = layer0_boundaries(oracle, 4000, 32, mb, gr)
    n0 = bounds[len(bounds) // 2]
    part, _ = S.build_batched(rows, mb, gr, stop_at=n0, threads=THREADS, seed=3)
    ix = abi.Index.from_graph(part.points, part.zero, part.upper, part.M, ef_search=part.ef_search, storage="bin")
    assert (ix.insert(rows[np.argsort(ids)][n0:]) == np.arange(n0, 4000)).all()
    _same_graph(ix, full)


def test_empty_bin_index_stays_bin_across_successive_inserts(abi):
    rows = _bits(3000, 23, 8)
    ix, _ = abi.Index.build(np.zeros((0, 23), np.float32), storage="bin")
    assert ix.info().storage == abi.STORAGE["bin"]
    from oracle import oracle as O

    g = O.Graph(np.zeros((0, 23), np.float32), np.zeros((0, 64), np.uint32), [], 32, 100)
    mb, gr = _schedule(0)
    for a, b in ((0, 1), (1, 2), (2, 40), (40, 41), (41, 700), (700, 3000)):  # across several capacity doublings
        assert (ix.insert(rows[a:b]) == np.arange(a, b)).all()
        g = S.insert_batched(g, rows[a:b], mb, gr, threads=THREADS)
        _same_graph(ix, g)


# dims: 16 (4-byte rows: the removal moves words), 37 / 300 (10- and 75-byte rows: bytes), 1100 (long rows)
@pytest.mark.parametrize("dim,M,kind", [(16, 16, "random10"), (37, 8, "random50"), (300, 16, "every_other"), (1100, 8, "random10")])
def test_remove_equals_the_statement(abi, oracle, dim, M, kind):
    n = 1200 if dim > 500 else 2000
    rows, q = _bits(n, dim, dim + M, q=40)
    ix, _ = abi.Index.build(rows, M=M, storage="bin", seed=3)
    p, z, u = ix.export_graph()
    g = R.O.Graph(p, z, u, M, 100)
    rng = np.random.default_rng(dim)
    pids = np.arange(0, n, 2, dtype=np.uint32) if kind == "every_other" else \
        rng.permutation(n)[:int(n * {"random10": 0.1, "random50": 0.5}[kind])].astype(np.uint32)
    want, want_ids = R.remove(g, pids)
    assert (ix.remove(pids) == want_ids).all()
    _same_graph(ix, want)
    ox = oracle.from_graph(want)
    _same_search(ix.search(q, ef_search=64, k=10), ox.search(q, ef_search=64, k=10, threads=THREADS))


# ---- 5. exact and range search -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [3, 128, 129, 300, 640, 768, 1024, 1025, 4100])
def test_exact_and_range_search_every_scan_cell(abi, oracle, dim):
    pts, q = _bits(2500, dim, 1, q=37)
    fq = datagen.uniform(13, dim, 2)
    ix = _flat(abi, pts)
    for qq in (q, fq):
        want = oracle.bruteforce(pts, qq, 10, threads=THREADS)
        _same_exact(ix.exact_search(qq, 10), *want)
    h = bin_ref.hamming(q, pts)
    ids, dist, _ = ix.exact_search(q, 10)
    assert (dist == np.take_along_axis(h, ids.astype(np.int64), axis=1)).all() and (dist[:, -1] == np.sort(h, axis=1)[:, 9]).all()
    radius = float(np.sort(h, axis=1)[:, 20].min())  # an integer radius: every row tied at it is a hit
    got = ix.range_search(q, radius)
    want = range_ref.range_search(oracle, pts, q, radius)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    assert int(got[0][-1]) == int((h <= radius).sum())


# ---- 6. sharded: bin shards, and bin mixed with f32 shards -------------------------------------------------------------------

def test_sharded_bin_and_mixed(abi, oracle):
    from tests import merge_statement as ms
    from tests.k1_dispatch import Cell
    from tests.k1_dispatch_bin import k1_cell
    from tests.test_gpu_sharded import Shard, Spec, _oracle_graph

    from instant_distance_b200 import sharded

    comm = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    specs = [Spec(1200, 100, "bin"), Spec(1000, 100, "f32"), Spec(900, 100, "bin", M=32)]
    shards, offset = [], 0
    for i, sp in enumerate(specs):
        rows = _bits(sp.n, sp.dim, 700 + i)  # 0/1 rows for every shard, so the f32 shard holds the same kind of points
        ix, local = abi.Index.build(rows, M=sp.M, ef_search=sp.ef, seed=40 + i, storage=sp.storage)
        gmap = sharded.global_id_map(local, offset)
        ix.set_id_map(gmap)
        shards.append(Shard(ix, _oracle_graph(oracle, ix, sp)[0], gmap, sp))
        offset += sp.n
    try:
        ef, k = 64, 20
        for q in (_bits(64, 100, 77), datagen.uniform(64, 100, 78)):
            got = abi.sharded_search_multi([sh.ix for sh in shards], comm, q, ef_search=ef, k=k)
            keys = []
            for i, sh in enumerate(shards):
                ids, dist, lens, cnt = sh.ox.search(q, ef_search=ef, k=k, counters=True, threads=THREADS)
                real = np.arange(k)[None, :] < np.minimum(lens, k)[:, None]
                kk = (np.ascontiguousarray(dist).view(np.uint32).astype(np.uint64) << np.uint64(32)) | \
                    sh.gmap[np.where(real, ids, 0)].astype(np.uint64)
                kk[~real] = np.uint64(ms.KEY_NONE)
                keys.append(kk)
                assert Cell(**sh.ix.last_kernel()) == k1_cell(sh.spec.dim, sh.spec.M, ef, sh.spec.n, sh.spec.storage), f"shard {i}"
                assert (sh.ix.last_counters(len(q)) == cnt).all(), f"shard {i}: per-layer counters differ"
            _same_search(got, ms.merge(np.stack(keys), k, "l2sq"))
    finally:
        for sh in shards:
            sh.ix.close()
        comm.close()


# ---- 7. save / load ----------------------------------------------------------------------------------------------------------

def test_save_load_and_save_again(abi, tmp_path):
    rows, q = _bits(3000, 100, 21, q=100)
    ix, _ = abi.Index.build(rows, storage="bin", seed=4)
    path = str(tmp_path / "bin.idx")
    ix.save(path)
    ld, off = abi.Index.load(path, dim=100, M=32, storage="bin")
    assert ld.info().storage == abi.STORAGE["bin"] and off == os.path.getsize(path)
    a, b = ix.export_graph(), ld.export_graph()
    assert a[0].tobytes() == b[0].tobytes() and (a[1] == b[1]).all() and all((x == y).all() for x, y in zip(a[2], b[2]))
    _same_search(ld.search(q, ef_search=100, k=10), ix.search(q, ef_search=100, k=10))
    _same_exact(ld.exact_search(q, 10), *ix.exact_search(q, 10)[:2])
    ld.save(str(tmp_path / "again.idx"))
    assert open(path, "rb").read() == open(str(tmp_path / "again.idx"), "rb").read()
    f32, _ = abi.Index.load(path, dim=100, M=32)  # the file holds the 0/1 rows as f32
    assert f32.info().storage == abi.STORAGE["f32"] and f32.export_graph()[0].tobytes() == a[0].tobytes()
    assert set(np.unique(a[0])) <= {0.0, 1.0} and np.signbit(a[0]).sum() == 0


# ---- 8. heavy ties: dims 4, 16 and 37, duplicate rows, the tie list and the retry pass ---------------------------------------

@pytest.mark.parametrize("dim", [4, 16, 37])
def test_heavy_ties_and_duplicates(abi, oracle, monkeypatch, dim):
    """Every row about 20 times over: most queries have tied distances at the ef boundary, where collect_ties decides.  Each ef
    also runs with 1024-slot visited tables, which send the queries to the retry pass (at dims 16 and 37; at dim 4, with 16
    distinct rows, a traversal visits too few ids to fill them)."""
    r = np.random.default_rng(dim)
    base = _bits(300, dim, 90 + dim)
    rows = base[r.integers(0, 300, 6000)]
    q = _bits(200, dim, 190 + dim)
    ix, _ = abi.Index.build(rows, storage="bin", seed=6)
    ox = _oracle(oracle, ix)
    for ef in (10, 100, 1024):
        want = ox.search(q, ef_search=ef, k=ef, threads=THREADS)
        _same_search(ix.search(q, ef_search=ef, k=ef), want)  # (a query that failed even the retry pass raises IDB_ERR_CAPACITY)
        d = want[1]
        assert ((np.diff(d, axis=1) == 0) & np.isfinite(d[:, 1:])).any(axis=1).mean() > 0.9
        with monkeypatch.context() as m:
            m.setenv("IDB_VIS_TIER", "0")
            m.setenv("IDB_VIS_SLOTS", "1024")
            small = _flat_graph(abi, ix)
            _same_search(small.search(q, ef_search=ef, k=ef), want)
            if ef >= 100 and dim > 4:
                assert small.last_retried(0xFFFFFFFF) > 0


def test_classes_of_2500_duplicates(abi, oracle):
    """dim 4 has 16 distinct 0/1 rows; 40 000 rows hold each about 2 500 times, more than ef 1024 plus the 1024-entry tie list.
    The build and the search must still equal the oracle.  (Selection by (distance, PointId) links the copies of a class to a
    small part of it, so a traversal meets only that part and its tie list does not overflow: DESIGN §3d.)"""
    rows = _bits(40000, 4, 404)
    assert np.unique(rows, axis=0).shape[0] == 16
    q = _bits(100, 4, 405)
    ix, _ = abi.Index.build(rows, storage="bin", seed=7)
    ox = _oracle(oracle, ix)
    for ef in (100, 1024):
        _same_search(ix.search(q, ef_search=ef, k=ef), ox.search(q, ef_search=ef, k=ef, threads=THREADS))


def _flat_graph(abi, ix):
    """The same graph and rows adopted again (picks up the visited-table settings of the environment)."""
    p, zero, upper = ix.export_graph()
    return abi.Index.from_graph(p, zero, upper, 32, storage="bin")


def test_build_that_overflows_the_retry_pass_fails_cleanly(abi, monkeypatch):
    """A bin build over duplicate rows with small visited tables for KA and its retry pass: IDB_ERR_CAPACITY, and no index."""
    for k, v in {"IDB_VIS_TIER": "0", "IDB_VIS_SLOTS": "1024", "IDB_RETRY_SLOTS": "1024"}.items():
        monkeypatch.setenv(k, v)
    base = _bits(64, 16, 55)
    rows = base[np.random.default_rng(1).integers(0, 64, 6000)]
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(rows, storage="bin", seed=9, ef_construction=200)
    assert e.value.status == abi.ERR_CAPACITY
    monkeypatch.delenv("IDB_RETRY_SLOTS")
    monkeypatch.delenv("IDB_VIS_SLOTS")
    ix, _ = abi.Index.build(rows[:2000], storage="bin", seed=9)  # the device is fine afterwards
    assert int(ix.info().n) == 2000


# ---- 9. the Python module ------------------------------------------------------------------------------------------------

def test_python_module_with_bin_storage(abi, oracle, tmp_path):
    import instant_distance as idist

    rows, q = _bits(2000, 64, 31, q=30)
    cfg = idist.Config()
    cfg.storage, cfg.seed = "bin", 9
    h, ids = idist.Hnsw.build(rows[:1500].tolist(), cfg)
    assert h._ix.info().storage == abi.STORAGE["bin"]
    g = h._ix.export_graph()
    assert g[0].tobytes() == rows[:1500][np.argsort(np.asarray(ids))].tobytes()
    ox = oracle.from_graph(oracle.Graph(g[0], g[1], g[2], 32, 100))
    _same_search(h.search_many(q, k=10), ox.search(q, ef_search=100, k=10, threads=THREADS))
    _same_exact(h.search_exact(q, k=10), *oracle.bruteforce(g[0], q, 10))
    got = h.search_range(q, 20.0)
    want = range_ref.range_search(oracle, g[0], q, 20.0)
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(got, want))
    assert h.insert(rows[1500:].tolist()) == list(range(1500, 2000))
    new_ids = h.remove([3, 5, 1999])
    assert int(h._ix.info().n) == 1997 and new_ids[4] == 3
    path = str(tmp_path / "m.idx")
    h.dump(path)
    ld = idist.Hnsw.load(path, dim=64, M=32, storage="bin")
    assert ld._ix.info().storage == abi.STORAGE["bin"]
    assert ld._ix.export_graph()[0].tobytes() == h._ix.export_graph()[0].tobytes()
    _same_search(ld.search_many(q, k=10), h.search_many(q, k=10))
    hm = idist.HnswMap.build(rows[:500].tolist(), [str(i) for i in range(500)], cfg)
    hm.remove([0])
    hm.dump(path)
    lm = idist.HnswMap.load(path, dim=64, M=32, storage="bin")
    assert lm.values == hm.values and lm._ix.info().storage == abi.STORAGE["bin"]
