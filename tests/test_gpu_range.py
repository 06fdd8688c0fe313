"""Exact range search (idb_range_search_batch_*): offsets, ids and distance BYTES equal to the CPU statement (tests/range_ref.py: the
full exact ordering of the oracle's brute force cut at the radius) over every scan cell, row type, metric, radius edge, capacity
outcome, index origin and entry point."""
import ctypes as C
import threading

import numpy as np
import pytest

from tests import datagen, range_ref
from tests.f16_ref import f16_round
from tests.q8_ref import roundtrip as q8_round

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF


def bf16_round(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u.astype(np.uint64) + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)


ROUND = {"f32": lambda x: np.ascontiguousarray(x, dtype=np.float32), "bf16": bf16_round, "f16": f16_round, "q8": q8_round}


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    return _abi


def flat(abi, pts, storage="f32", metric="l2sq"):
    """An index over `pts` with an empty graph: the range search reads the rows only."""
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    zero = np.full((pts.shape[0], 4), INVALID, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage, metric=metric)


def assert_same(got, want):
    for g, w, what in zip(got, want, ("offsets", "ids", "distances")):
        assert g.dtype == w.dtype and g.shape == w.shape, what
        assert g.tobytes() == w.tobytes(), what


def raw(abi, ix, q, radius, capacity):
    """The host entry as it is: (status, offsets, ids, dist) with ids / dist of `capacity` entries."""
    q = ix._queries(q)
    offsets = np.full(q.shape[0] + 1, 7, dtype=np.uint64)
    ids = np.full(max(capacity, 1), 7, dtype=np.uint32)
    dist = np.full(max(capacity, 1), 7, dtype=np.float32)
    st = abi.lib().idb_range_search_batch_f32(ix._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.shape[0], float(radius), capacity,
                                              offsets.ctypes.data_as(C.POINTER(C.c_uint64)), ids.ctypes.data_as(C.POINTER(C.c_uint32)),
                                              dist.ctypes.data_as(C.POINTER(C.c_float)))
    return st, offsets, ids, dist


def radii(order_dist, ranks=(0, 9, 99)):
    """Radii that give about `rank` + 1 hits per query: the median over the queries of that neighbour's distance."""
    return [float(np.median(order_dist[:, min(r, order_dist.shape[1] - 1)])) for r in ranks]


def check(abi, oracle, ix, stored, q, radius_list=None, metric="l2sq", id_map=None):
    ids, dist = range_ref.full_order(oracle, stored, q, metric)
    for r in radius_list if radius_list is not None else radii(dist):
        assert_same(ix.range_search(q, r), range_ref.cut(ids, dist, r, id_map))


@pytest.mark.parametrize("dim", [1, 3, 4, 127, 128, 129, 300, 640, 768, 1024, 1025, 4100])
def test_every_scan_cell(abi, oracle, dim):
    pts = datagen.uniform(2500, dim, 1)  # 3 slices of 834 rows at this query count, the last one ragged
    q = datagen.uniform(37, dim, 2)
    check(abi, oracle, flat(abi, pts), pts, q)


@pytest.mark.parametrize("storage", ["f32", "bf16", "f16", "q8"])
@pytest.mark.parametrize("dim", [3, 300, 1025])
def test_row_types_against_the_stored_rows(abi, oracle, storage, dim):
    pts = datagen.sift_shaped(2000, dim, 3)
    q = datagen.sift_shaped(29, dim, 4)
    check(abi, oracle, flat(abi, pts, storage), ROUND[storage](pts), q)


@pytest.mark.parametrize("storage", ["f32", "bf16", "f16", "q8"])
def test_cosine_with_zero_rows_and_queries(abi, oracle, storage):
    pts = datagen.uniform(3000, 100, 5) - 0.5
    pts[[0, 7, 1500, 2999]] = 0.0
    q = datagen.uniform(41, 100, 6) - 0.5
    q[[0, 40]] = 0.0
    stored = ROUND[storage](abi.normalize(pts))
    ix = flat(abi, stored, storage, metric="cosine")
    _, d = range_ref.full_order(oracle, stored, q, "cosine")
    check(abi, oracle, ix, stored, q, radii(d) + [0.5, 0.0], metric="cosine")  # 0.5: every zero row of a non-zero query


def test_ties_at_the_radius_and_duplicates_at_zero(abi, oracle):
    pts = datagen.grid_ties(20011, 3, 19, side=4)  # integer grid: many equal distances
    dup = pts[5].copy()
    for b in (0, 1000, 1001, 1002, 5004, 10009, 20010):  # the same row at and around slice boundaries
        pts[b] = dup
    q = np.concatenate([dup[None, :], datagen.grid_ties(20, 3, 20, side=4)]).astype(np.float32)
    ix = flat(abi, pts)
    check(abi, oracle, ix, pts, q, [0.0, 1.0, 2.0, 3.0])
    offsets, ids, dist = ix.range_search(q[:1], 0.0)
    assert offsets[1] >= 8 and (dist == 0).all() and (ids == np.sort(ids)).all()


def test_radius_edges(abi, oracle):
    pts = datagen.uniform(3000, 20, 21)
    pts[12, 3] = np.nan  # NaN distance to every query: never a hit
    pts[11] = 1e20       # +inf distance: a hit at radius +inf only
    q = datagen.uniform(9, 20, 22)
    ix = flat(abi, pts)
    ids, dist = range_ref.full_order(oracle, pts, q)
    edges = [-1.0, -0.0, 0.0, np.inf, float(np.finfo(np.float32).max)]
    hit = dist[3, 17]  # one ulp either side of a hit's distance
    edges += [float(np.nextafter(hit, np.float32(-np.inf))), float(hit), float(np.nextafter(hit, np.float32(np.inf)))]
    for r in edges:
        assert_same(ix.range_search(q, r), range_ref.cut(ids, dist, r))
    counts = [int(ix.range_search(q, r)[0][4]) for r in edges[-3:]]
    assert counts[0] < counts[1] <= counts[2]
    offsets, _, _ = ix.range_search(q, np.inf)
    assert (np.diff(offsets) == 2999).all()  # every row but the NaN one
    offsets, _, _ = ix.range_search(q, -1.0)
    assert (offsets == 0).all()


def test_no_hits_and_every_row_a_hit_ragged_slices(abi, oracle):
    pts = datagen.uniform(20011, 48, 17)  # a few queries: ~20 slices of 1001 rows, the last one shorter
    q = np.concatenate([datagen.uniform(4, 48, 18), np.full((1, 48), 100.0, np.float32)])  # the last query is far from every row
    ix = flat(abi, pts)
    ids, dist = range_ref.full_order(oracle, pts, q)
    for r in (float(dist[:4, 0].max()), 1000.0, float(dist[:, -1].max())):
        assert_same(ix.range_search(q, r), range_ref.cut(ids, dist, r))
    offsets, _, _ = ix.range_search(q, 1000.0)
    assert (np.diff(offsets)[:4] == 20011).all() and offsets[5] == offsets[4]


@pytest.mark.parametrize("nq", [1, 33, 1000])
def test_query_counts(abi, oracle, nq):
    pts = datagen.uniform(4000, 64, 13)
    check(abi, oracle, flat(abi, pts), pts, datagen.uniform(nq, 64, 14))


def test_capacity(abi, oracle):
    pts = datagen.uniform(3000, 16, 31)
    q = datagen.uniform(25, 16, 32)
    ix = flat(abi, pts)
    ids, dist = range_ref.full_order(oracle, pts, q)
    r = radii(dist, (40,))[0]
    want = range_ref.cut(ids, dist, r)
    total = int(want[0][-1])
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
    assert_same(ix.range_search(q, r, capacity=total), want)
    assert_same(ix.range_search(q, np.inf), range_ref.cut(ids, dist, np.inf))  # 75 000 hits: the binding's first guess is too small
    with pytest.raises(abi.IdbError) as e:
        ix.range_search(q, r, capacity=total - 1)
    assert e.value.status == abi.ERR_CAPACITY


def test_id_map_ties_ordered_by_point_id(abi, oracle):
    pts = datagen.grid_ties(5000, 3, 23, side=3)
    q = datagen.grid_ties(15, 3, 24, side=3)
    gmap = (np.arange(5000, dtype=np.uint32)[::-1] + 10).astype(np.uint32)  # reverses the PointId order
    ix = flat(abi, pts)
    ix.set_id_map(gmap)
    check(abi, oracle, ix, pts, q, [0.0, 1.0, 2.0], id_map=gmap)


def test_empty_and_one_point_index(abi, oracle):
    q = datagen.uniform(3, 8, 11)
    offsets, ids, dist = flat(abi, np.zeros((0, 8), np.float32)).range_search(q, np.inf)
    assert offsets.tobytes() == np.zeros(4, np.uint64).tobytes() and ids.size == 0 and dist.size == 0
    one = datagen.uniform(1, 8, 12)
    check(abi, oracle, flat(abi, one), one, q, [-1.0, 0.0, 0.5, np.inf])


def test_adopted_loaded_and_inserted_indexes(abi, oracle, tmp_path):
    pts = datagen.sift_shaped(5000, 40, 25)
    q = datagen.sift_shaped(50, 40, 26)
    built, _ = abi.Index.build(pts[:3000], seed=3)
    built.insert(pts[3000:])
    stored, zero, upper = built.export_graph()
    adopted = abi.Index.from_graph(stored, zero, upper, 32)
    path = str(tmp_path / "g.idx")
    built.save(path)
    loaded, _ = abi.Index.load(path, dim=40, M=32)
    ids, dist = range_ref.full_order(oracle, stored, q)
    rs = radii(dist)
    for ix in (built, adopted, loaded):
        for r in rs:
            assert_same(ix.range_search(q, r), range_ref.cut(ids, dist, r))


def test_prefix_of_the_exact_search(abi, oracle):
    pts = datagen.sift_shaped(6000, 32, 27)
    q = datagen.sift_shaped(200, 32, 28)
    ix = flat(abi, pts)
    e_ids, e_dist, _ = ix.exact_search(q, 1024)
    checked = 0
    for r in radii(e_dist, (0, 9, 99, 999)):
        offsets, ids, dist = ix.range_search(q, r)
        for i in range(q.shape[0]):
            c = int(offsets[i + 1] - offsets[i])
            if c > 1024:
                continue
            s = slice(int(offsets[i]), int(offsets[i + 1]))
            assert (ids[s] == e_ids[i, :c]).all() and dist[s].tobytes() == e_dist[i, :c].tobytes()
            assert c == 1024 or not e_dist[i, c] <= r
            checked += 1
    assert checked > 500


def test_identical_calls_give_identical_bytes(abi):
    pts = datagen.grid_ties(30000, 4, 29, side=5)  # many ties: the append order differs between runs, the output may not
    q = datagen.grid_ties(300, 4, 30, side=5)
    ix = flat(abi, pts)
    a = ix.range_search(q, 3.0)
    b = ix.range_search(q, 3.0)
    assert a[0][-1] > 100000
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_device_entry_unaligned_on_every_lane(abi, oracle):
    import torch

    n, dim, nq = 3000, 30, 45
    pts = datagen.uniform(n, dim, 33)
    q = datagen.uniform(nq, dim, 34)
    ix = flat(abi, pts)
    ids, dist = range_ref.full_order(oracle, pts, q)
    r = radii(dist, (30,))[0]
    want = range_ref.cut(ids, dist, r)
    total = int(want[0][-1])
    buf = torch.zeros(nq * dim + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(q.ravel()).cuda()  # 4-byte aligned rows of 30 floats
    torch.cuda.synchronize()
    for lane in range(abi.lib().idb_index_num_lanes()):
        offsets = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
        d_ids = torch.empty(total, dtype=torch.int32, device="cuda")
        d_dist = torch.empty(total, dtype=torch.float32, device="cuda")
        got = ix.range_search_device(buf.data_ptr() + 4, nq, r, total, offsets.data_ptr(), d_ids.data_ptr(), d_dist.data_ptr(),
                                     lane=lane)
        assert got == total
        assert_same((offsets.cpu().numpy().view(np.uint64), d_ids.cpu().numpy().view(np.uint32), d_dist.cpu().numpy()), want)
        offsets.fill_(7)
        with pytest.raises(abi.IdbError) as e:
            ix.range_search_device(buf.data_ptr() + 4, nq, r, total - 1, offsets.data_ptr(), d_ids.data_ptr(), d_dist.data_ptr(),
                                   lane=lane)
        assert e.value.status == abi.ERR_CAPACITY and f"(total {total})" in str(e.value)
        assert offsets.cpu().numpy().view(np.uint64).tobytes() == want[0].tobytes()


def test_range_exact_and_approximate_searches_at_once(abi):
    pts = datagen.sift_shaped(6000, 64, 35)
    q = datagen.sift_shaped(400, 64, 36)
    ix, _ = abi.Index.build(pts, seed=5)
    want_approx = ix.search(q, ef_search=64, k=10)
    kernel, fetches = ix.last_kernel(), ix.last_full_fetches()
    want_exact = ix.exact_search(q, 10)
    r = float(np.median(want_exact[1][:, 9]))
    want_range = ix.range_search(q, r)
    assert ix.last_kernel() == kernel and ix.last_full_fetches() == fetches  # the diagnostics still describe the approximate search
    bad = []

    def run(fn, want):
        for _ in range(5):
            got = fn()
            if not all(np.array_equal(a, b) for a, b in zip(got, want)):
                bad.append(fn)

    ts = [threading.Thread(target=run, args=(lambda: ix.range_search(q, r), want_range)),
          threading.Thread(target=run, args=(lambda: ix.range_search(q[::-1], r), ix.range_search(q[::-1], r))),
          threading.Thread(target=run, args=(lambda: ix.exact_search(q, 10), want_exact)),
          threading.Thread(target=run, args=(lambda: ix.search(q, ef_search=64, k=10), want_approx))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not bad


def test_python_module_search_range(abi, oracle):
    import instant_distance as idist

    rows = datagen.sift_shaped(1500, 24, 37)
    q = datagen.sift_shaped(20, 24, 38)
    cfg = idist.Config()
    cfg.seed = 1
    h, _ = idist.Hnsw.build(rows.tolist(), cfg)
    stored = h._ix.export_graph()[0]
    ids, dist = range_ref.full_order(oracle, stored, q)
    r = radii(dist, (20,))[0]
    want = range_ref.cut(ids, dist, r)
    assert_same(h.search_range(q, r), want)
    assert_same(h.search_range(q.tolist(), r), want)
    hm = idist.HnswMap.build(rows.tolist(), [str(i) for i in range(1500)], cfg)
    stored = hm._ix.export_graph()[0]
    ids, dist = range_ref.full_order(oracle, stored, q)
    assert_same(hm.search_range(q, r), range_ref.cut(ids, dist, r))
