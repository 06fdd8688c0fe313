"""GPU inserts (idb_index_insert_f32) against the CPU statement of the insert (tests/insert_statement.py), bit for bit.

Continuation: a statement graph stopped at a layer-0 batch boundary n0, adopted on the GPU, plus a GPU insert of the remaining rows,
is the full batched build.  The other cases insert into GPU-built, loaded and empty indexes, several times in a row, one row at a
time, under every visited flavour and through KA's retry pass; then search, exact search, save / load and export must agree with
the oracle on the statement's graph.  Also: the refusals that need an index, the capacity failure (and what the Python module and
the C++ mirror keep after it), a shard with an id map, concurrent searches, the Python module and the recall an insert gives up.
"""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from tests import cosine_ref, datagen
from tests import insert_statement as S
from tests.test_insert_statement import (RECALL_EF, RECALL_GAP, RECALL_N0, layer0_boundaries, recall_at_10, recall_case)

pytestmark = pytest.mark.gpu
THREADS = min(32, os.cpu_count() or 8)


def bf16_round(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((u.astype(np.uint64) + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(np.float32)


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _schedule(insert_batch):
    if insert_batch:
        return insert_batch, 8
    return (max(1, int(os.environ.get("IDB_BUILD_MAXBATCH", "16384"))), max(1, int(os.environ.get("IDB_BUILD_GROWTH", "8"))))


def _same(ix, g):
    p, zero, upper = ix.export_graph()
    assert p.shape == g.points.shape and p.tobytes() == g.points.tobytes(), "stored rows differ"
    bad = np.nonzero((zero != g.zero).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} zero rows differ, first PointId {bad[0]}: gpu {zero[bad[0]].tolist()} statement {g.zero[bad[0]].tolist()}"
    assert len(upper) == len(g.upper)
    for a, b in zip(upper, g.upper):
        assert a.shape == b.shape and (a == b).all()


def _adopt(abi, g, storage="f32", metric="l2sq"):
    return abi.Index.from_graph(g.points, g.zero, g.upper, g.M, ef_search=g.ef_search, storage=storage, metric=metric)


# ---- continuation: stopped statement graph + GPU insert == full batched build ------------------------------------------------

CONTINUATION = [
    # (gen, n, dim, params, insert_batch, storage, metric)
    (datagen.uniform, 3000, 16, {}, 0, "f32", "l2sq"),
    (datagen.uniform, 3000, 16, {}, 7, "f32", "l2sq"),
    (datagen.uniform, 3000, 16, {}, 64, "f32", "l2sq"),
    (datagen.uniform, 2000, 37, {"M": 4}, 0, "f32", "l2sq"),
    (datagen.sift_shaped, 4000, 128, {}, 0, "f32", "l2sq"),
    (datagen.uniform, 2000, 300, {"M": 64}, 0, "f32", "l2sq"),
    (datagen.uniform, 1000, 1100, {"M": 16}, 0, "f32", "l2sq"),
    (datagen.uniform, 3000, 16, {"heuristic": 0}, 0, "f32", "l2sq"),
    (datagen.uniform, 3000, 24, {"keep_pruned": 0}, 0, "f32", "l2sq"),
    (datagen.sift_shaped, 4000, 128, {}, 0, "bf16", "l2sq"),
    (datagen.sift_shaped, 3000, 64, {}, 0, "f32", "cosine"),
    (datagen.sift_shaped, 3000, 64, {}, 0, "bf16", "cosine"),
]


@pytest.mark.parametrize("gen,n,dim,kw,insert_batch,storage,metric", CONTINUATION)
def test_continuation_is_the_full_build(abi, oracle, gen, n, dim, kw, insert_batch, storage, metric):
    rows = gen(n, dim, 40 + dim)
    stored = cosine_ref.normalize(oracle, rows) if metric == "cosine" else rows
    stored = bf16_round(stored) if storage == "bf16" else stored
    mb, gr = _schedule(insert_batch)
    kw = dict(kw, seed=3)
    full, ids = S.build_batched(stored, mb, gr, threads=THREADS, **kw)
    bounds = layer0_boundaries(oracle, n, kw.get("M", 32), mb, gr)
    n0 = bounds[len(bounds) // 2]
    part, _ = S.build_batched(stored, mb, gr, stop_at=n0, threads=THREADS, **kw)
    ix = _adopt(abi, part, storage=storage, metric=metric)
    # the caller's rows of PointIds [n0, n): the insert normalises and narrows them as the build did
    orig = rows[np.argsort(ids)][n0:]
    new_ids = ix.insert(orig, insert_batch=insert_batch, **{k: v for k, v in kw.items() if k != "seed"})
    assert (new_ids == np.arange(n0, n)).all()
    _same(ix, full)


# ---- against the statement's insert ------------------------------------------------------------------------------------------

def _stmt_insert(g, rows, insert_batch=0, **kw):
    mb, gr = _schedule(insert_batch)
    return S.insert_batched(g, rows, mb, gr, threads=THREADS, **kw)


def _graph(ix, M, ef=100):
    from oracle import oracle as O

    p, z, u = ix.export_graph()
    return O.Graph(p, z, u, M, ef)


def test_insert_into_gpu_built_and_loaded_index(abi, oracle, tmp_path):
    rows = datagen.sift_shaped(6000, 128, 7)
    ix, _ = abi.Index.build(rows[:3000], seed=2)
    g = _graph(ix, 32)
    want = _stmt_insert(g, rows[3000:])
    ix.insert(rows[3000:])
    _same(ix, want)
    path = str(tmp_path / "a.idx")
    ix0, _ = abi.Index.build(rows[:3000], seed=2)
    ix0.save(path)
    ld, _ = abi.Index.load(path, dim=128, M=32)
    ld.insert(rows[3000:])
    _same(ld, want)


@pytest.mark.parametrize("storage", ["f32", "bf16"])
def test_insert_into_empty_index_then_successive_inserts(abi, oracle, storage):
    rows = datagen.uniform(5000, 24, 8)
    ix, _ = abi.Index.build(np.zeros((0, 24), np.float32), storage=storage)
    stored = bf16_round(rows) if storage == "bf16" else rows
    empty = oracle.Graph(np.zeros((0, 24), np.float32), np.zeros((0, 64), np.uint32), [], 32, 100)
    g = empty
    # sizes that cross several capacity doublings, and single rows
    for a, b in ((0, 1), (1, 2), (2, 40), (40, 41), (41, 700), (700, 5000)):
        ids = ix.insert(rows[a:b])
        assert (ids == np.arange(a, b)).all()
        g = _stmt_insert(g, stored[a:b])
        _same(ix, g)
    assert int(ix.info().n) == 5000


@pytest.mark.parametrize("tier", ["0", "1", "2"])
def test_visited_tiers(abi, oracle, monkeypatch, tier):
    monkeypatch.setenv("IDB_VIS_TIER", tier)
    rows = datagen.uniform(6000, 32, 9)
    ix, _ = abi.Index.build(rows[:2000], seed=5)
    want = _stmt_insert(_graph(ix, 32), rows[2000:])
    ix.insert(rows[2000:])
    _same(ix, want)


def test_retry_pass_and_b16_demotion(abi, oracle, monkeypatch):
    monkeypatch.setenv("IDB_B16_BYTES", "2048")
    monkeypatch.setenv("IDB_B16_CAP", "4")
    rows = datagen.uniform(8000, 16, 10)
    ix, _ = abi.Index.build(rows[:2000], seed=6, ef_construction=200)
    want = _stmt_insert(_graph(ix, 32), rows[2000:], ef_construction=200)
    ix.insert(rows[2000:], ef_construction=200)
    _same(ix, want)


def test_n_crosses_a_b16_injectivity_boundary(abi, oracle, monkeypatch):
    """b16 ids are exact while ceil(n / 32768) <= buckets; the 8-bucket tables of IDB_B16_BYTES=512 serve n <= 262144 only.  The
    index is built below that bound and the insert takes it above: the insert's traversals see n = n0 + m for the whole call, so
    none of its batches can use the b16 flavour the build could."""
    monkeypatch.setenv("IDB_B16_BYTES", "512")
    rows = datagen.uniform(270_000, 4, 11)
    kw = dict(M=2, ml=0.5, ef_construction=16)
    ix, _ = abi.Index.build(rows[:250_000], seed=7, **kw)
    want = _stmt_insert(_graph(ix, 2), rows[250_000:], **kw)
    ix.insert(rows[250_000:], M=2, ef_construction=16)
    _same(ix, want)


# ---- after an insert: search, exact search, save / load, export ---------------------------------------------------------------

@pytest.mark.parametrize("screen", ["1", "0"])
def test_search_after_insert(abi, oracle, monkeypatch, tmp_path, screen):
    monkeypatch.setenv("IDB_SCREEN", screen)
    rows = datagen.sift_shaped(8000, 128, 12)
    q = datagen.sift_shaped(300, 128, 13)
    ix, _ = abi.Index.build(rows[:4000], seed=8)
    want = _stmt_insert(_graph(ix, 32), rows[4000:])
    ix.insert(rows[4000:])
    o = oracle.from_graph(want)
    ids, dist, lens = ix.search(q, ef_search=100, k=10)
    cnt = ix.last_counters(len(q))
    o_ids, o_dist, o_lens, o_cnt = o.search(q, ef_search=100, k=10, counters=True)
    assert (ids == o_ids).all() and dist.tobytes() == o_dist.tobytes() and (lens == o_lens).all()
    assert (cnt == o_cnt).all()
    e_ids, e_dist, _ = ix.exact_search(q, k=10)
    b_ids, b_dist = oracle.bruteforce(want.points, q, 10)
    assert (e_ids == b_ids).all() and e_dist.tobytes() == b_dist.tobytes()
    path = str(tmp_path / "b.idx")
    ix.save(path)
    ld, _ = abi.Index.load(path, dim=128, M=32)
    l_ids, l_dist, l_lens = ld.search(q, ef_search=100, k=10)
    assert (l_ids == ids).all() and l_dist.tobytes() == dist.tobytes() and (l_lens == lens).all()
    _same(ld, want)


# ---- refusals that need an index ----------------------------------------------------------------------------------------------

def test_refusals(abi):
    rows = datagen.uniform(500, 8, 14)
    ix, _ = abi.Index.build(rows, seed=1, M=16)
    h = ix._h
    L = abi.lib()
    p = abi.default_params(M=16)
    r = abi.f32(rows[:3])
    ids = np.empty(3, np.uint32)
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), 3, 9, C.byref(p), None, abi.ptr(ids, C.c_uint32)) == abi.ERR_INVALID_ARG
    p32 = abi.default_params(M=32)
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), 3, 8, C.byref(p32), None, abi.ptr(ids, C.c_uint32)) == abi.ERR_INVALID_ARG
    g = np.arange(3, dtype=np.uint32)
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), 3, 8, C.byref(p), abi.ptr(g, C.c_uint32), None) == abi.ERR_INVALID_ARG
    big = 0xFFFFFFFF - 500
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), big, 8, C.byref(p), None, None) == abi.ERR_INVALID_ARG
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), 0, 8, C.byref(p), None, None) == abi.OK
    ix.set_id_map(np.arange(500, dtype=np.uint32) + 7)
    assert L.idb_index_insert_f32(h, abi.ptr(r, C.c_float), 3, 8, C.byref(p), None, None) == abi.ERR_INVALID_ARG
    assert int(ix.info().n) == 500


# ---- capacity failure ---------------------------------------------------------------------------------------------------------

# A 1024-slot hash set for KA (IDB_VIS_TIER=0, IDB_VIS_SLOTS=1024) and for its retry pass (IDB_RETRY_SLOTS=1024): an insert whose
# traversal visits more than 3/4 of the slots overflows both, which the insert reports as IDB_ERR_CAPACITY (a host-side report).
# Inserting into a 500-point index, the first batches cannot visit that many ids (a batch at g0 sees g0 points); with
# ef_construction = 200 later ones do.
SMALL_TABLES = {"IDB_VIS_TIER": "0", "IDB_VIS_SLOTS": "1024", "IDB_RETRY_SLOTS": "1024"}


def _capacity_case():
    rows = datagen.uniform(6000, 16, 15)
    return rows[:500], rows[500:]


def _boundaries(n0, n1):
    mb, gr = _schedule(0)
    out, g0 = [], n0
    while g0 < n1:
        out.append(g0)
        g0 += min(mb, max(1, g0 // gr), n1 - g0)
    return out


def test_capacity_failure_keeps_the_batches_before_it(abi, oracle, monkeypatch):
    """The index keeps the batches before the failing one, equals the statement stopped there, still searches correctly and takes
    further inserts."""
    for k, v in SMALL_TABLES.items():
        monkeypatch.setenv(k, v)
    base, more = _capacity_case()
    ix, _ = abi.Index.build(base, seed=9, ef_construction=200)
    g = _graph(ix, 32)
    seen = []
    with pytest.raises(abi.IdbError) as e:
        ix.insert(more, ef_construction=200, progress=lambda d, t: seen.append(d))
    assert e.value.status == abi.ERR_CAPACITY
    n = int(ix.info().n)
    assert 500 < n < 6000 and n in _boundaries(500, 6000), "n must be the failing batch's first PointId"
    assert seen and seen[-1] == n - 500  # progress reported the batches that stand
    want = _stmt_insert(g, more[:n - 500], ef_construction=200)
    _same(ix, want)
    q = datagen.uniform(100, 16, 17)
    ids, dist, lens = ix.search(q, ef_search=50, k=10)
    o_ids, o_dist, o_lens = oracle.from_graph(want).search(q, ef_search=50, k=10)
    assert (ids == o_ids).all() and dist.tobytes() == o_dist.tobytes() and (lens == o_lens).all()
    monkeypatch.delenv("IDB_RETRY_SLOTS")
    ix2 = _adopt(abi, want)  # with a full-size retry pass the same rows go in, from where the failure left the index
    assert (ix2.insert(more[n - 500:], ef_construction=200) == np.arange(n, 6000)).all()
    _same(ix2, _stmt_insert(want, more[n - 500:], ef_construction=200))


def test_progress_reports_m_once(abi):
    rows = datagen.uniform(3000, 8, 19)
    ix, _ = abi.Index.build(rows[:1000], seed=1)
    seen = []
    ix.insert(rows[1000:], progress=lambda d, t: seen.append((d, t)))
    assert seen[-1] == (2000, 2000) and [d for d, _ in seen].count(2000) == 1
    assert all(a[0] < b[0] for a, b in zip(seen, seen[1:]))
    empty, _ = abi.Index.build(np.zeros((0, 8), np.float32))
    seen.clear()
    empty.insert(rows[:1], progress=lambda d, t: seen.append((d, t)))
    assert seen == [(1, 1)]


def test_python_module_after_a_failed_insert(abi, monkeypatch, tmp_path):
    """A failed HnswMap.insert keeps one value per PointId the index kept: searches return them and dump / load round-trips."""
    import instant_distance as idm

    for k, v in SMALL_TABLES.items():
        monkeypatch.setenv(k, v)
    base, more = _capacity_case()
    cfg = idm.Config()
    cfg.seed = 9
    cfg.ef_construction = 200
    h = idm.HnswMap.build(base.tolist(), [f"b{i}" for i in range(500)], cfg)
    with pytest.raises(Exception) as e:
        h.insert(more.tolist(), [f"d{i}" for i in range(5500)], cfg)
    assert getattr(e.value, "status", None) == abi.ERR_CAPACITY
    n = int(h._ix.info().n)
    assert 500 < n < 6000 and len(h.values) == n and h.values[-1] == f"d{n - 501}"
    s = idm.Search()
    h.search(more[n - 501].tolist(), s)
    first = next(iter(s))
    assert first.pid == n - 1 and first.value == f"d{n - 501}" and first.distance == 0.0
    path = str(tmp_path / "f.idx")
    h.dump(path)
    h2 = idm.HnswMap.load(path, dim=16, M=32)
    assert h2.values == h.values


def test_cpp_mirror_after_a_failed_insert(abi, tmp_path):
    import subprocess

    from tests.conftest import ROOT

    libdir = os.path.join(ROOT, "instant-distance_b200", "lib")
    exe = str(tmp_path / "test_hpp_insert")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cpp", "test_hpp_insert.cpp"),
                           "-L" + libdir, "-linstant_distance_b200", "-Wl,-rpath," + libdir])
    r = subprocess.run([exe], env=dict(os.environ, **SMALL_TABLES), capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr


# ---- shard with an id map -----------------------------------------------------------------------------------------------------

def test_shard_with_id_map(abi, oracle):
    from tests import merge_statement as MS

    rows = datagen.sift_shaped(4000, 32, 18)
    q = datagen.sift_shaped(100, 32, 19)
    ix, _ = abi.Index.build(rows[:2000], seed=10)
    gid = np.arange(2000, dtype=np.uint32) * 3 + 1
    ix.set_id_map(gid)
    new_gid = np.arange(2000, dtype=np.uint32) * 3 + 6001
    want = _stmt_insert(_graph(ix, 32), rows[2000:])
    with pytest.raises(abi.IdbError):
        ix.insert(rows[2000:])  # the map needs the new rows' global ids
    ix.insert(rows[2000:], global_ids=new_gid)
    _same(ix, want)
    gmap = np.concatenate([gid, new_gid])
    comm = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    try:
        ids, dist, lens = ix.sharded_search(comm, q, ef_search=64, k=10)
    finally:
        comm.close()
    o_ids, o_dist, o_lens = oracle.from_graph(want).search(q, ef_search=64, k=64)
    keys = np.full((1, len(q), 64), MS.KEY_NONE, dtype=np.uint64)
    for i in range(len(q)):
        for j in range(int(o_lens[i])):
            keys[0, i, j] = (int(o_dist[i, j].view(np.uint32)) << 32) | int(gmap[o_ids[i, j]])
    m_ids, m_dist, m_lens = MS.report(MS.merged_keys(keys, 10))
    assert (ids == m_ids).all() and dist.tobytes() == m_dist.tobytes() and (lens == m_lens).all()


# ---- concurrency --------------------------------------------------------------------------------------------------------------

def test_searches_see_the_index_before_or_after_the_insert(abi):
    rows = datagen.sift_shaped(60_000, 64, 20)
    q = datagen.sift_shaped(500, 64, 21)
    ix, _ = abi.Index.build(rows[:30_000], seed=11)
    before = ix.search(q, ef_search=64, k=10)
    results, errors = [], []
    stop = threading.Event()

    def searcher():
        try:
            while not stop.is_set():
                results.append(ix.search(q, ef_search=64, k=10))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=searcher) for _ in range(2)]
    for t in th:
        t.start()
    ix.insert(rows[30_000:])
    stop.set()
    for t in th:
        t.join()
    after = ix.search(q, ef_search=64, k=10)
    assert not errors
    assert results
    for r in results:
        same_before = all((a == b).all() for a, b in zip(r, before))
        same_after = all((a == b).all() for a, b in zip(r, after))
        assert same_before or same_after


# ---- the Python module --------------------------------------------------------------------------------------------------------

def test_python_module(abi, tmp_path):
    import instant_distance as idm

    cfg = idm.Config()
    cfg.seed = 5
    pts = [list(map(float, r)) for r in datagen.uniform(300, 6, 22)]
    more = [list(map(float, r)) for r in datagen.uniform(50, 6, 23)]
    h = idm.HnswMap.build(pts, [f"v{i}" for i in range(300)], cfg)
    new = h.insert(more[:-1] + [more[-1][:4]], [f"w{i}" for i in range(50)])
    assert new == list(range(300, 350))
    assert h.values[300:] == [f"w{i}" for i in range(50)]
    s = idm.Search()
    h.search(more[3], s)
    first = next(iter(s))
    assert first.pid == 303 and first.value == "w3" and first.distance == 0.0
    with pytest.raises(TypeError, match="point array too long"):
        h.insert([[0.0] * 7], ["x"])
    path = str(tmp_path / "m.idx")
    h.dump(path)
    h2 = idm.HnswMap.load(path, dim=6, M=32)
    assert h2.values == h.values
    h2.search(more[3], s)
    assert next(iter(s)).pid == 303
    plain, _ = idm.Hnsw.build(pts, cfg)
    assert plain.insert(more) == list(range(300, 350))


# ---- recall -------------------------------------------------------------------------------------------------------------------

def test_recall_within_the_calibrated_gap(abi, oracle):
    pts, q = recall_case(oracle)
    full, _ = abi.Index.build(pts, seed=1)
    grown, _ = abi.Index.build(pts[:RECALL_N0], seed=1)
    grown.insert(pts[RECALL_N0:])
    r = {}
    for name, ix in (("full", full), ("inserted", grown)):
        truth = ix.exact_search(q, k=10)[0]
        r[name] = recall_at_10(ix.search(q, ef_search=RECALL_EF, k=10)[0], truth)
    print(r)
    assert r["inserted"] >= r["full"] - RECALL_GAP
