"""GPU removals (idb_index_remove) against the CPU statement of the removal (tests/remove_ref.py), bit for bit.

Each case exports the index before the call (the rows as stored, widened exactly; the zero and upper rows), states the removal on
that graph, and compares the index after the call with it: rows, zero rows, upper rows, layer counts and new ids.  The cases cover
dims on both sides of each CH boundary and the long-row kernel, M 4 to 64, ef_construction below 2M and 1024, the four storages,
cosine, simple mode, keep_pruned 0 and 1, the staged K2 cells, and removal sets from one point to all of them; on GPU-built,
sequentially built, adopted (with repeated ids in a row), loaded, inserted-into indexes and a shard with an id map.  On the result,
the graph search, the exact and range searches, a later insert and save / load agree with the oracle; searches on other threads see
the index before or after the call; the Python module and the C++ mirror agree with the ABI; and the recall stays within the gap
tests/test_remove_cpu.py calibrates on the CPU.
"""
import os
import subprocess
import threading

import numpy as np
import pytest

from tests import datagen
from tests import insert_statement as S
from tests import range_ref
from tests import remove_ref as R
from tests.test_remove_cpu import RECALL_EF, RECALL_GAP, recall_at_10, recall_case

pytestmark = pytest.mark.gpu
THREADS = min(32, os.cpu_count() or 8)
INVALID = R.INVALID


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _graph(ix, M, ef=100):
    p, z, u = ix.export_graph()
    return R.O.Graph(p, z, u, M, ef)


def _same(ix, g):
    p, zero, upper = ix.export_graph()
    assert p.shape == g.points.shape and p.tobytes() == g.points.tobytes(), "stored rows differ"
    bad = np.nonzero((zero != g.zero).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} zero rows differ, first PointId {bad[0]}: gpu {zero[bad[0]].tolist()} statement {g.zero[bad[0]].tolist()}"
    assert [u.shape[0] for u in upper] == [u.shape[0] for u in g.upper], "layer counts differ"
    for l, (a, b) in enumerate(zip(upper, g.upper)):
        assert (a == b).all(), f"layer {l + 1} differs"


def _pids(kind, g, rng):
    n = g.points.shape[0]
    if kind == "one":
        return np.array([n // 3], np.uint32)
    if kind == "pid0":
        return np.array([0], np.uint32)
    if kind == "hub":
        deg = np.bincount(g.zero[g.zero != INVALID].astype(np.int64), minlength=n)
        return np.array([int(np.argmax(deg))], np.uint32)
    if kind == "top_layer":
        return np.arange(g.upper[-1].shape[0], dtype=np.uint32)
    if kind == "every_other":
        return np.arange(0, n, 2, dtype=np.uint32)
    if kind == "neighbours":  # every candidate of the last point's row: its neighbours and theirs
        p = n - 1
        ring = set(g.zero[p][g.zero[p] != INVALID].tolist())
        for r in list(ring):
            ring.update(g.zero[r][g.zero[r] != INVALID].tolist())
        ring.discard(p)
        return np.array(sorted(ring), np.uint32)
    share = {"random10": 0.1, "random50": 0.5}[kind]
    return rng.permutation(n)[:int(n * share)].astype(np.uint32)  # in no particular order


def _check(abi, ix, g, pids, **kw):
    """Removes pids from ix (whose exported graph is g) and compares with the statement; returns the statement's graph and new ids."""
    want, want_ids = R.remove(g, pids, **kw)
    new_ids = ix.remove(pids, **kw)
    assert (new_ids == want_ids).all()
    _same(ix, want)
    return want, want_ids


# (dim, M, ef_construction, storage, metric, heuristic, keep_pruned, removal)
CASES = [
    (16, 16, 100, "f32", "l2sq", 1, 1, "random10"),
    (37, 4, 6, "bf16", "l2sq", 1, 0, "random50"),       # ef_construction < 2M: the cap binds
    (128, 32, 100, "f32", "l2sq", 1, 1, "one"),
    (129, 16, 1024, "f16", "cosine", 1, 1, "every_other"),
    (256, 8, 40, "q8", "l2sq", 1, 1, "hub"),
    (257, 8, 40, "f32", "l2sq", 0, 1, "random10"),       # simple mode
    (300, 32, 100, "bf16", "cosine", 1, 0, "pid0"),
    (384, 8, 64, "f16", "l2sq", 1, 1, "random50"),
    (385, 8, 64, "q8", "cosine", 1, 1, "random10"),
    (768, 8, 64, "f32", "l2sq", 1, 1, "top_layer"),
    (1024, 8, 64, "bf16", "l2sq", 0, 1, "random10"),
    (1100, 8, 100, "f32", "l2sq", 1, 1, "random50"),     # long rows
    (24, 8, 50, "f32", "l2sq", 1, 1, "neighbours"),      # an empty row
    (64, 64, 200, "f32", "l2sq", 1, 1, "random50"),      # M = 64: rows of thousands of candidates
]


@pytest.mark.parametrize("dim,M,efc,storage,metric,heuristic,keep_pruned,kind", CASES)
def test_remove_matches_the_statement(abi, dim, M, efc, storage, metric, heuristic, keep_pruned, kind):
    n = 1200 if dim > 500 or M == 64 else 2000
    rows = datagen.sift_shaped(n, dim, dim + M)
    ix, _ = abi.Index.build(rows, M=M, ef_construction=efc, storage=storage, metric=metric, seed=3)
    g = _graph(ix, M)
    pids = _pids(kind, g, np.random.default_rng(dim))
    want, want_ids = _check(abi, ix, g, pids, ef_construction=efc, heuristic=heuristic, keep_pruned=keep_pruned)
    if kind == "neighbours":
        assert (want.zero[want_ids[n - 1]] == INVALID).all()
    if kind == "top_layer":
        assert len(want.upper) == len(g.upper) - 1


@pytest.mark.parametrize("dim", [128, 300])
def test_staged_cells(abi, monkeypatch, dim):
    monkeypatch.setenv("IDB_BUILD_STAGE", "1")
    rows = datagen.sift_shaped(2000, dim, 4)
    ix, _ = abi.Index.build(rows, M=16, seed=4)
    g = _graph(ix, 16)
    _check(abi, ix, g, _pids("random10", g, np.random.default_rng(1)))


def test_sequentially_built_and_adopted_with_repeated_ids(abi):
    rows = datagen.sift_shaped(1500, 32, 5)
    ix, _ = abi.Index.build(rows, M=8, insert_batch=1, seed=5)
    g = _graph(ix, 8)
    _check(abi, ix, g, _pids("random10", g, np.random.default_rng(2)))
    zero = g.zero.copy()
    for r in range(0, zero.shape[0], 7):  # repeat the first entry of every 7th row in its last slot
        if zero[r, 0] != INVALID:
            zero[r, -1] = zero[r, 0]
    adopted = abi.Index.from_graph(g.points, zero, g.upper, 8)
    g2 = R.O.Graph(g.points, zero, g.upper, 8, 100)
    _check(abi, adopted, g2, _pids("random50", g2, np.random.default_rng(3)))


def test_loaded_and_inserted_into(abi, tmp_path):
    rows = datagen.sift_shaped(3000, 128, 6)
    ix, _ = abi.Index.build(rows[:2000], seed=6)
    ix.insert(rows[2000:])
    g = _graph(ix, 32)
    path = str(tmp_path / "a.idx")
    ix.save(path)
    _check(abi, ix, g, _pids("random10", g, np.random.default_rng(4)))
    ld, _ = abi.Index.load(path, dim=128, M=32)
    _check(abi, ld, g, _pids("every_other", g, None))


def test_all_points_then_insert(abi):
    rows = datagen.sift_shaped(1500, 40, 7)
    ix, _ = abi.Index.build(rows[:1000], M=8, storage="bf16", seed=7)
    g = _graph(ix, 8)
    _check(abi, ix, g, np.arange(1000, dtype=np.uint32)[::-1].copy())
    info = ix.info()
    assert int(info.n) == 0 and int(info.n_layers) == 0 and int(info.dim) == 40 and int(info.storage) == 1
    assert int(ix.search(rows[:3], ef_search=10, k=5)[2].max()) == 0
    fresh, _ = abi.Index.build(np.zeros((0, 40), np.float32), M=8, storage="bf16")
    for a, b in ((1000, 1001), (1001, 1500)):
        ix.insert(rows[a:b], M=8)
        fresh.insert(rows[a:b], M=8)
    _same(ix, _graph(fresh, 8))


def test_refusals_leave_the_index_as_it_was(abi):
    rows = datagen.sift_shaped(500, 16, 8)
    ix, _ = abi.Index.build(rows, M=8, seed=8)
    g = _graph(ix, 8)
    for pids, msg in (([3, 500], "pids\\[1\\] = 500"), ([3, 9, 3], "pids\\[2\\] = 3 repeats pids\\[0\\]")):
        with pytest.raises(abi.IdbError, match=msg):
            ix.remove(np.array(pids, np.uint32))
    with pytest.raises(abi.IdbError, match="M = 16 differs"):
        ix.remove(np.array([1], np.uint32), M=16)
    _same(ix, g)
    assert (ix.remove(np.zeros(0, np.uint32)) == np.arange(500)).all()
    _same(ix, g)


# ---- the searches, an insert and save / load on the result --------------------------------------------------------------------------

def test_searches_insert_and_save_after_a_removal(abi, oracle, tmp_path):
    rows = datagen.sift_shaped(5000, 96, 9)
    q = datagen.sift_shaped(300, 96, 10)
    ix, _ = abi.Index.build(rows[:4000], seed=9)
    g = _graph(ix, 32)
    want, _ = _check(abi, ix, g, _pids("random10", g, np.random.default_rng(5)))
    ids, dist, lens, = ix.search(q, ef_search=64, k=10)
    cnt = ix.last_counters(len(q))
    o_ids, o_dist, o_lens, o_cnt = oracle.from_graph(want).search(q, ef_search=64, k=10, counters=True)
    assert (ids == o_ids).all() and dist.tobytes() == o_dist.tobytes() and (lens == o_lens).all()
    assert (cnt == o_cnt).all()
    e_ids, e_dist, _ = ix.exact_search(q, k=10)
    b_ids, b_dist = oracle.bruteforce(want.points, q, 10, threads=THREADS)
    assert (e_ids == b_ids).all() and e_dist.tobytes() == b_dist.tobytes()
    radius = float(np.median(b_dist[:, 4]))
    off, r_ids, r_dist = ix.range_search(q, radius)
    w_off, w_ids, w_dist = range_ref.range_search(oracle, want.points, q, radius)
    assert (off == w_off).all() and (r_ids == w_ids).all() and r_dist.tobytes() == w_dist.tobytes()
    path = str(tmp_path / "r.idx")
    ix.save(path)
    ld, _ = abi.Index.load(path, dim=96, M=32)
    _same(ld, want)
    mb, gr = S.schedule(0)
    grown = S.insert_batched(want, rows[4000:], mb, gr, threads=THREADS)
    ix.insert(rows[4000:])
    _same(ix, grown)


def test_shard_with_id_map(abi, oracle):
    rows = datagen.sift_shaped(2000, 32, 11)
    q = datagen.sift_shaped(50, 32, 12)
    ix, _ = abi.Index.build(rows, M=16, seed=11)
    gid = np.arange(2000, dtype=np.uint32) * 5 + 3
    ix.set_id_map(gid)
    g = _graph(ix, 16)
    _, new_ids = _check(abi, ix, g, _pids("random10", g, np.random.default_rng(6)))
    kept_gid = gid[new_ids != INVALID]
    e_ids, _, _ = ix.exact_search(q, k=10)
    b_ids, _ = oracle.bruteforce(g.points[new_ids != INVALID], q, 10, threads=THREADS)
    assert (e_ids == kept_gid[b_ids]).all()


# ---- concurrency ------------------------------------------------------------------------------------------------------------------

def test_searches_see_the_index_before_or_after_the_removal(abi):
    rows = datagen.sift_shaped(60_000, 64, 13)
    q = datagen.sift_shaped(500, 64, 14)
    ix, _ = abi.Index.build(rows, seed=12)
    before = ix.search(q, ef_search=64, k=10)
    results, errors = [], []
    stop = threading.Event()

    def searcher():
        try:
            while not stop.is_set():
                results.append(ix.search(q, ef_search=64, k=10))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=searcher) for _ in range(4)]
    for t in th:
        t.start()
    ix.remove(np.arange(0, 60_000, 4, dtype=np.uint32))
    stop.set()
    for t in th:
        t.join()
    after = ix.search(q, ef_search=64, k=10)
    assert not errors and results
    for r in results:
        same_before = all((a == b).all() for a, b in zip(r, before))
        same_after = all((a == b).all() for a, b in zip(r, after))
        assert same_before or same_after


# ---- the Python module and the C++ mirror ---------------------------------------------------------------------------------------------

def test_python_module(abi, tmp_path):
    import instant_distance as idm

    cfg = idm.Config()
    cfg.seed = 5
    pts = [list(map(float, r)) for r in datagen.uniform(400, 6, 15)]
    h = idm.HnswMap.build(pts, [f"v{i}" for i in range(400)], cfg)
    vals = list(h.values)
    raw = abi.Index.build(np.array(pts, np.float32), **cfg._params())[0]
    gone = list(range(0, 400, 3))
    new_ids = h.remove(gone)
    assert new_ids == [int(x) for x in raw.remove(np.array(gone, np.uint32))]
    _same(h._ix, _graph(raw, 32))
    assert h.values == [v for x, v in enumerate(vals) if x % 3]
    path = str(tmp_path / "m.idx")
    h.dump(path)
    assert idm.HnswMap.load(path, dim=6, M=32).values == h.values
    plain, _ = idm.Hnsw.build(pts, cfg)
    assert plain.remove(gone) == new_ids


def test_cpp_mirror(abi, tmp_path):
    from tests.conftest import ROOT

    libdir = os.path.join(ROOT, "instant-distance_b200", "lib")
    exe = str(tmp_path / "test_hpp_remove")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cpp", "test_hpp_remove.cpp"),
                           "-L" + libdir, "-linstant_distance_b200", "-Wl,-rpath," + libdir])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr


# ---- recall -------------------------------------------------------------------------------------------------------------------------

def test_recall_within_the_calibrated_gap(abi, oracle):
    rows, q, pids = recall_case()
    ix, _ = abi.Index.build(rows, seed=1)
    ix.remove(pids)
    survivors = ix.export_graph()[0]
    fresh, fresh_ids = abi.Index.build(survivors, seed=1)
    row_of = np.empty_like(fresh_ids)
    row_of[fresh_ids] = np.arange(fresh_ids.size, dtype=np.uint32)
    truth, _ = oracle.bruteforce(survivors, q, 10, threads=THREADS)
    r_removed = recall_at_10(ix.search(q, ef_search=RECALL_EF, k=10)[0], truth)
    r_fresh = recall_at_10(row_of[fresh.search(q, ef_search=RECALL_EF, k=10)[0]], truth)
    print(f"recall@10 fresh build {r_fresh:.4f}  after removal {r_removed:.4f}")
    assert r_removed >= r_fresh - RECALL_GAP
