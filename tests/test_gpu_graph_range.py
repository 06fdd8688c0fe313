"""Graph range search (idb_graph_range_search_batch_*): offsets, ids and distance BYTES equal to the CPU statement
(tests/graph_range_ref.py: the oracle's search of the same graph for the seeds, a worklist closure over the exported layer 0, the
exact range statement's distances) over every expansion cell, row type, metric, M, ef, radius edge, capacity outcome, retry path, index
origin and entry point; and the relations to the exact range search that the definition implies."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from tests import datagen, graph_range_ref, range_ref
from tests.golden.make_golden import case_inputs

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    return _abi


def assert_same(got, want):
    for g, w, what in zip(got, want, ("offsets", "ids", "distances")):
        assert g.dtype == w.dtype and g.shape == w.shape, what
        assert g.tobytes() == w.tobytes(), what


def radii(order_dist, ranks=(0, 9, 99)):
    """Radii that give about `rank` + 1 exact hits per query: the median over the queries of that neighbour's distance."""
    return [float(np.median(order_dist[:, min(r, order_dist.shape[1] - 1)])) for r in ranks]


def reference(oracle, ix, q, radius_list, ef=0, id_map=None):
    """The statement's results at each radius, on the index's exported graph (rows as stored)."""
    info = ix.info()
    stored, zero, upper = ix.export_graph()
    full = range_ref.full_order(oracle, stored, q, ix.metric)
    ef = ef or int(info.ef_search)
    return [graph_range_ref.graph_range_search(oracle, stored, zero, upper, int(info.M), q, r, ef, ix.metric, id_map, full=full)
            for r in radius_list], full


def check(abi, oracle, ix, q, radius_list=None, ef=0, id_map=None):
    if radius_list is None:
        stored = ix.export_graph()[0]
        radius_list = radii(range_ref.full_order(oracle, stored, q, ix.metric)[1])
    want, full = reference(oracle, ix, q, radius_list, ef, id_map)
    for r, w in zip(radius_list, want):
        assert_same(ix.graph_range_search(q, r, ef_search=ef), w)
    return want, full


def raw(abi, ix, q, radius, capacity, ef=0):
    """The host entry as it is: (status, offsets, ids, dist) with ids / dist of `capacity` entries."""
    q = ix._queries(q)
    offsets = np.full(q.shape[0] + 1, 7, dtype=np.uint64)
    ids = np.full(max(capacity, 1), 7, dtype=np.uint32)
    dist = np.full(max(capacity, 1), 7, dtype=np.float32)
    st = abi.lib().idb_graph_range_search_batch_f32(ix._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.shape[0], ef, float(radius),
                                                    capacity, offsets.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                    ids.ctypes.data_as(C.POINTER(C.c_uint32)), dist.ctypes.data_as(C.POINTER(C.c_float)))
    return st, offsets, ids, dist


def ring_index(abi, pts, M=4, extra_seed=0, **kw):
    """An adopted graph whose layer 0 is strongly connected: a ring, plus a few random links per row."""
    n = pts.shape[0]
    zero = np.full((n, 2 * M), INVALID, dtype=np.uint32)
    ring = np.arange(n, dtype=np.uint32)
    zero[:, 0], zero[:, 1] = np.roll(ring, 1), np.roll(ring, -1)
    rng = np.random.default_rng(extra_seed)
    for p in range(n):
        extra = rng.choice(n, size=min(M, n), replace=False)
        extra = [int(x) for x in extra if x != p and x not in zero[p, :2]][: 2 * M - 2]
        zero[p, 2:2 + len(extra)] = extra
    return abi.Index.from_graph(pts, zero, [], M, **kw)


@pytest.mark.parametrize("dim", [16, 128, 129, 256, 257, 384, 385, 512, 513, 640, 641, 768, 769, 1024, 1025])
def test_every_expansion_cell(abi, oracle, dim):
    pts = datagen.sift_shaped(1500, dim, 1)
    q = datagen.sift_shaped(40, dim, 2)
    ix, _ = abi.Index.build(pts, seed=1, M=16, ef_construction=64)
    check(abi, oracle, ix, q, ef=40)


@pytest.mark.parametrize("storage", ["f32", "bf16", "f16", "q8", "bin"])
@pytest.mark.parametrize("dim", [20, 200, 300, 500, 700, 900, 1025])  # CH 1, 2, 3, 4, 6, 8 and long rows
def test_row_types_against_the_stored_rows(abi, oracle, storage, dim):
    pts = datagen.sift_shaped(1200, dim, 3)
    q = datagen.sift_shaped(30, dim, 4)
    if storage == "bin":
        med = np.median(pts, axis=0)
        pts, q = (pts > med).astype(np.float32), (q > med).astype(np.float32)
    ix, _ = abi.Index.build(pts, seed=2, M=16, ef_construction=64, storage=storage)
    check(abi, oracle, ix, q, ef=32)


@pytest.mark.parametrize("storage", ["f32", "bf16", "f16", "q8"])
def test_cosine_with_zero_rows_and_queries(abi, oracle, storage):
    pts = datagen.uniform(2000, 100, 5) - 0.5
    pts[[0, 7, 1500, 1999]] = 0.0
    q = datagen.uniform(41, 100, 6) - 0.5
    q[[0, 40]] = 0.0
    ix, _ = abi.Index.build(pts, seed=3, M=16, ef_construction=64, storage=storage, metric="cosine")
    stored = ix.export_graph()[0]
    _, d = range_ref.full_order(oracle, stored, q, "cosine")
    check(abi, oracle, ix, q, radii(d) + [0.5, 0.0, np.inf], ef=50)  # 0.5: every zero row of a non-zero query


@pytest.mark.parametrize("M", [16, 32, 64])
@pytest.mark.parametrize("ef", [1, 0, 1024])
def test_m_and_ef(abi, oracle, M, ef):
    pts = datagen.sift_shaped(2500, 24, 7)
    q = datagen.sift_shaped(50, 24, 8)
    ix, _ = abi.Index.build(pts, seed=4, M=M, ef_construction=80)
    check(abi, oracle, ix, q, ef=ef)


def test_radius_edges(abi, oracle):
    pts = datagen.uniform(3000, 20, 21)
    pts[12, 3] = np.nan  # NaN distance to every query: never a hit
    pts[11] = 1e20       # +inf distance: a hit at radius +inf only
    pts[[100, 2000, 2999]] = pts[50]  # duplicates across rows: radius 0 from a copy finds them all
    q = np.concatenate([pts[50:51], datagen.uniform(9, 20, 22)]).astype(np.float32)
    ix = ring_index(abi, pts, M=8)
    ids, dist = range_ref.full_order(oracle, pts, q)
    hit = dist[3, 17]
    edges = [-1.0, -0.0, 0.0, float(np.nextafter(hit, np.float32(-np.inf))), float(hit), float(np.nextafter(hit, np.float32(np.inf))),
             float(np.finfo(np.float32).max), np.inf]
    check(abi, oracle, ix, q, edges, ef=64)
    counts = [int(ix.graph_range_search(q, r, ef_search=64)[0][4]) for r in edges[3:6]]
    assert counts[0] <= counts[1] <= counts[2]
    offsets, got_ids, _ = ix.graph_range_search(q[:1], 0.0, ef_search=64)
    assert 0 < got_ids.size and set(got_ids.tolist()) <= {50, 100, 2000, 2999}
    assert_same(ix.graph_range_search(q, np.inf, ef_search=64), range_ref.cut(ids, dist, np.inf))  # connected: the exact result
    offsets, _, _ = ix.graph_range_search(q, -1.0, ef_search=64)
    assert (offsets == 0).all()


def test_heavy_ties_golden_graph(abi, oracle):
    z = np.load(os.path.join(GOLDEN, "grid_ties_1500x3_M32.npz"))
    from tests.golden.make_golden import SEARCH_CASES

    case = [c for c in SEARCH_CASES if c[0] == "grid_ties_1500x3_M32"][0]
    _, gen, n, dim, M, _, _, _ = case
    pts, q = case_inputs(gen, n, dim)
    p = np.empty_like(pts)
    p[z["ids_map"]] = pts
    upper = [z[f"upper{i}"] for i in range(int(z["n_upper"]))]
    ix = abi.Index.from_graph(p, z["zero"], upper, M)
    check(abi, oracle, ix, q, [0.0, 1.0, 2.0, 5.0], ef=10)
    check(abi, oracle, ix, q, [0.0, 1.0, 2.0, 5.0], ef=100)


def test_subsequence_of_the_exact_range_search_and_monotone(abi, oracle):
    pts = datagen.sift_shaped(20000, 32, 27)
    q = datagen.sift_shaped(1000, 32, 28)
    ix, _ = abi.Index.build(pts, seed=5)
    e_ids, e_dist, _ = ix.exact_search(q, 1000)
    rs = radii(e_dist, (0, 9, 99, 999))
    want, _ = reference(oracle, ix, q, rs)
    prev = None
    for r, w in zip(rs, want):
        got = ix.graph_range_search(q, r)
        assert_same(got, w)
        exact = ix.range_search(q, r)
        counts = np.diff(got[0])
        for i in range(q.shape[0]):
            gi, gd = got[1][got[0][i]:got[0][i + 1]], got[2][got[0][i]:got[0][i + 1]]
            ei, ed = exact[1][exact[0][i]:exact[0][i + 1]], exact[2][exact[0][i]:exact[0][i + 1]]
            pos = np.searchsorted(ei, gi, sorter=np.argsort(ei))
            idx = np.argsort(ei)[pos]
            assert (ei[idx] == gi).all() and (np.diff(idx) > 0).all() and gd.tobytes() == ed[idx].tobytes()
        if prev is not None:
            assert (counts >= prev).all()
        prev = counts
    assert prev.sum() > 0


def test_capacity(abi, oracle):
    pts = datagen.sift_shaped(3000, 16, 31)
    q = datagen.sift_shaped(25, 16, 32)
    ix, _ = abi.Index.build(pts, seed=6)
    _, d = range_ref.full_order(oracle, pts, q)
    r = radii(d, (40,))[0]
    (want,), _ = reference(oracle, ix, q, [r])
    total = int(want[0][-1])
    assert total > 100
    st, offsets, got_ids, got_dist = raw(abi, ix, q, r, total)  # exactly at capacity
    assert st == abi.OK
    assert_same((offsets, got_ids, got_dist), want)
    st, offsets, got_ids, got_dist = raw(abi, ix, q, r, total - 1)  # one over
    assert st == abi.ERR_CAPACITY and offsets.tobytes() == want[0].tobytes()
    assert (got_ids == 7).all() and (got_dist == 7).all()  # nothing else written
    st, offsets, got_ids, got_dist = raw(abi, ix, q, r, int(offsets[-1]))  # the re-call, sized exactly
    assert st == abi.OK
    assert_same((offsets, got_ids, got_dist), want)
    st, offsets, _, _ = raw(abi, ix, q, r, 0)  # a counting call
    assert st == abi.ERR_CAPACITY and offsets.tobytes() == want[0].tobytes()
    st, offsets, _, _ = raw(abi, ix, q, -1.0, 0)
    assert st == abi.OK and (offsets == 0).all()
    with pytest.raises(abi.IdbError) as e:
        ix.graph_range_search(q, r, capacity=total - 1)
    assert e.value.status == abi.ERR_CAPACITY


@pytest.mark.parametrize("scratch", ["1", "24"])
def test_the_retry_pass_gives_the_same_bytes(abi, oracle, monkeypatch, scratch):
    pts = datagen.sift_shaped(6000, 40, 41)
    q = datagen.sift_shaped(300, 40, 42)
    ix, _ = abi.Index.build(pts, seed=7, M=16)
    stored, zero, upper = ix.export_graph()
    monkeypatch.setenv("IDB_GRAPH_RANGE_SCRATCH", scratch)  # read when an index is created: the main pass holds `scratch` hits
    forced = abi.Index.from_graph(stored, zero, upper, 16)
    monkeypatch.delenv("IDB_GRAPH_RANGE_SCRATCH")
    _, d = range_ref.full_order(oracle, stored, q)
    rs = radii(d, (0, 9, 99, 999))
    want, _ = reference(oracle, ix, q, rs, ef=64)
    for r, w in zip(rs, want):
        assert_same(ix.graph_range_search(q, r, ef_search=64), w)
        assert_same(forced.graph_range_search(q, r, ef_search=64), w)


def test_id_map_reversing_point_id_order(abi, oracle):
    pts = datagen.grid_ties(5000, 3, 23, side=6)
    q = datagen.grid_ties(15, 3, 24, side=6)
    ix, _ = abi.Index.build(pts, seed=8)
    gmap = (np.arange(5000, dtype=np.uint32)[::-1] + 10).astype(np.uint32)
    ix.set_id_map(gmap)
    check(abi, oracle, ix, q, [0.0, 1.0, 2.0, 4.0], ef=64, id_map=gmap)


def test_empty_and_one_point_index(abi, oracle):
    q = datagen.uniform(3, 8, 11)
    empty = abi.Index.from_graph(np.zeros((0, 8), np.float32), np.zeros((0, 4), np.uint32), [], 2)
    offsets, ids, dist = empty.graph_range_search(q, np.inf)
    assert offsets.tobytes() == np.zeros(4, np.uint64).tobytes() and ids.size == 0 and dist.size == 0
    one = datagen.uniform(1, 8, 12)
    ix = abi.Index.from_graph(one, np.full((1, 4), INVALID, np.uint32), [], 2)
    check(abi, oracle, ix, q, [-1.0, 0.0, 0.5, np.inf], ef=10)
    offsets, ids, _ = ix.graph_range_search(q, np.inf)
    assert (np.diff(offsets) == 1).all() and (ids == 0).all()


def test_inserted_removed_adopted_and_loaded_indexes(abi, oracle, tmp_path):
    pts = datagen.sift_shaped(5000, 40, 25)
    q = datagen.sift_shaped(50, 40, 26)
    built, _ = abi.Index.build(pts[:3000], seed=3)
    built.insert(pts[3000:])
    check(abi, oracle, built, q, ef=48)
    stored, zero, upper = built.export_graph()
    adopted = abi.Index.from_graph(stored, zero, upper, 32)
    check(abi, oracle, adopted, q, ef=48)
    path = str(tmp_path / "g.idx")
    built.save(path)
    loaded, _ = abi.Index.load(path, dim=40, M=32)
    check(abi, oracle, loaded, q, ef=48)
    built.remove(np.arange(0, 5000, 7, dtype=np.uint32))
    check(abi, oracle, built, q, ef=48)


def test_device_entry_unaligned_on_every_lane(abi, oracle):
    import torch

    n, dim, nq = 3000, 30, 45
    pts = datagen.sift_shaped(n, dim, 33)
    q = datagen.sift_shaped(nq, dim, 34)
    ix, _ = abi.Index.build(pts, seed=9)
    _, d = range_ref.full_order(oracle, pts, q)
    r = radii(d, (30,))[0]
    (want,), _ = reference(oracle, ix, q, [r], ef=40)
    total = int(want[0][-1])
    buf = torch.zeros(nq * dim + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(q.ravel()).cuda()  # 4-byte aligned rows of 30 floats
    torch.cuda.synchronize()
    for lane in range(abi.lib().idb_index_num_lanes()):
        offsets = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
        d_ids = torch.empty(total, dtype=torch.int32, device="cuda")
        d_dist = torch.empty(total, dtype=torch.float32, device="cuda")
        got = ix.graph_range_search_device(buf.data_ptr() + 4, nq, r, total, offsets.data_ptr(), d_ids.data_ptr(), d_dist.data_ptr(),
                                           ef_search=40, lane=lane)
        assert got == total
        assert_same((offsets.cpu().numpy().view(np.uint64), d_ids.cpu().numpy().view(np.uint32), d_dist.cpu().numpy()), want)
        offsets.fill_(7)
        with pytest.raises(abi.IdbError) as e:
            ix.graph_range_search_device(buf.data_ptr() + 4, nq, r, total - 1, offsets.data_ptr(), d_ids.data_ptr(), d_dist.data_ptr(),
                                         ef_search=40, lane=lane)
        assert e.value.status == abi.ERR_CAPACITY and f"(total {total})" in str(e.value)
        assert offsets.cpu().numpy().view(np.uint64).tobytes() == want[0].tobytes()


def test_identical_calls_give_identical_bytes(abi):
    pts = datagen.grid_ties(30000, 4, 29, side=5)  # many ties: the append order differs between runs, the output may not
    q = datagen.grid_ties(300, 4, 30, side=5)
    ix, _ = abi.Index.build(pts, seed=10)
    a = ix.graph_range_search(q, 3.0)
    b = ix.graph_range_search(q, 3.0)
    assert a[0][-1] > 10000
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_the_seed_search_counts_as_a_plain_search(abi):
    pts = datagen.sift_shaped(6000, 64, 43)
    q = datagen.sift_shaped(200, 64, 44)
    ix, _ = abi.Index.build(pts, seed=11)
    ix.search(q, ef_search=80, k=80)
    want = (ix.last_counters(200), ix.last_kernel(), ix.last_full_fetches(), ix.last_retried(0xFFFFFFFF))
    ix.exact_search(q, 5)  # something else in between
    ix.graph_range_search(q, 1e30, ef_search=80)
    got = (ix.last_counters(200), ix.last_kernel(), ix.last_full_fetches(), ix.last_retried(0xFFFFFFFF))
    assert (got[0] == want[0]).all() and got[1:] == want[1:]
    assert all(ix.last_failures(lane) == 0 for lane in range(abi.lib().idb_index_num_lanes()))


def test_graph_range_exact_range_exact_and_approximate_searches_at_once(abi):
    pts = datagen.sift_shaped(6000, 64, 35)
    q = datagen.sift_shaped(400, 64, 36)
    ix, _ = abi.Index.build(pts, seed=5)
    want_approx = ix.search(q, ef_search=64, k=10)
    want_exact = ix.exact_search(q, 10)
    r = float(np.median(want_exact[1][:, 9]))
    want_range = ix.range_search(q, r)
    want_graph = ix.graph_range_search(q, r, ef_search=64)
    bad = []

    def run(fn, want):
        for _ in range(5):
            got = fn()
            if not all(np.array_equal(a, b) for a, b in zip(got, want)):
                bad.append(fn)

    ts = [threading.Thread(target=run, args=(lambda: ix.graph_range_search(q, r, ef_search=64), want_graph)),
          threading.Thread(target=run, args=(lambda: ix.range_search(q, r), want_range)),
          threading.Thread(target=run, args=(lambda: ix.exact_search(q, 10), want_exact)),
          threading.Thread(target=run, args=(lambda: ix.search(q, ef_search=64, k=10), want_approx))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not bad


def test_python_module_search_range_graph(abi, oracle):
    import instant_distance as idist

    rows = datagen.sift_shaped(1500, 24, 37)
    q = datagen.sift_shaped(20, 24, 38)
    cfg = idist.Config()
    cfg.seed = 1
    h, _ = idist.Hnsw.build(rows.tolist(), cfg)
    stored = h._ix.export_graph()[0]
    _, d = range_ref.full_order(oracle, stored, q)
    r = radii(d, (20,))[0]
    (want,), _ = reference(oracle, h._ix, q, [r])
    assert_same(h.search_range_graph(q, r), want)
    assert_same(h.search_range_graph(q.tolist(), r), want)
    (want,), _ = reference(oracle, h._ix, q, [r], ef=30)
    assert_same(h.search_range_graph(q, r, ef_search=30), want)
    hm = idist.HnswMap.build(rows.tolist(), [str(i) for i in range(1500)], cfg)
    (want,), _ = reference(oracle, hm._ix, q, [r])
    assert_same(hm.search_range_graph(q, r), want)
