"""Exact k-NN (idb_exact_search_batch_*): ids, distance BYTES and lengths bit for bit equal to the CPU brute force of the canonical
distance (oracle.bruteforce, tests/cosine_ref.bruteforce; ties by lower PointId, NaN last) over every row type, metric, kernel
instantiation (CH cells and the long-row kernel), slice layout and query chunking."""
import os
import threading

import numpy as np
import pytest

from tests import cosine_ref, datagen

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF


def bf16_round(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((u.astype(np.uint64) + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(np.float32)


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    return _abi


def flat(abi, pts, storage="f32", metric="l2sq"):
    """An index over `pts` with an empty graph: the exact search reads the rows only."""
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    zero = np.full((pts.shape[0], 4), INVALID, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage, metric=metric)


def assert_same(got, want_ids, want_dist):
    ids, dist, lens = got
    k = want_ids.shape[1]
    assert ids.shape == want_ids.shape
    assert (ids == want_ids).all()
    assert dist.tobytes() == np.ascontiguousarray(want_dist, dtype=np.float32).tobytes()
    assert (lens == (want_ids != INVALID).sum(1)).all() and (lens <= k).all()


def check_l2(abi, oracle, pts, q, k, storage="f32"):
    ix = flat(abi, pts, storage)
    ref = bf16_round(pts) if storage == "bf16" else pts
    want = oracle.bruteforce(ref, q, k, threads=os.cpu_count() or 1)
    assert_same(ix.exact_search(q, k), *want)
    return ix


@pytest.mark.parametrize("dim", [1, 3, 4, 127, 128, 129, 300, 640, 768, 1024, 1025, 4100])
def test_f32_every_kernel_cell(abi, oracle, dim):
    pts = datagen.uniform(2500, dim, 1)  # 3 slices of 834 rows, the last one ragged
    q = datagen.uniform(37, dim, 2)
    check_l2(abi, oracle, pts, q, 10)


@pytest.mark.parametrize("dim", [3, 128, 300, 768, 1025])
def test_bf16_rows_equal_the_oracle_on_rounded_rows(abi, oracle, dim):
    pts = datagen.sift_shaped(2500, dim, 3)
    q = datagen.sift_shaped(29, dim, 4)
    check_l2(abi, oracle, pts, q, 10, storage="bf16")


@pytest.mark.parametrize("storage", ["f32", "bf16"])
def test_cosine_with_zero_rows_and_queries(abi, oracle, storage):
    pts = datagen.uniform(3000, 100, 5) - 0.5
    pts[[0, 7, 1500, 2999]] = 0.0
    q = datagen.uniform(41, 100, 6) - 0.5
    q[[0, 40]] = 0.0
    stored = abi.normalize(pts)
    if storage == "bf16":
        stored = bf16_round(stored)
    ix = flat(abi, stored, storage, metric="cosine")
    want_ids, want_dist = oracle.bruteforce(stored, cosine_ref.normalize(oracle, q), 20)
    assert_same(ix.exact_search(q, 20), want_ids, cosine_ref.reported(want_dist))
    if storage == "f32":  # the stored rows are the canonical normalisation: the CPU statement from the raw rows agrees
        assert_same(ix.exact_search(q, 20), *cosine_ref.bruteforce(oracle, pts, q, 20))


@pytest.mark.parametrize("k", [1, 10, 100, 1024])
def test_k(abi, oracle, k):
    pts = datagen.uniform(3000, 16, 7)
    q = datagen.uniform(53, 16, 8)
    check_l2(abi, oracle, pts, q, k)


def test_k_above_n_pads(abi, oracle):
    pts = datagen.uniform(50, 24, 9)
    q = datagen.uniform(5, 24, 10)
    ix = check_l2(abi, oracle, pts, q, 100)
    ids, dist, lens = ix.exact_search(q, 100)
    assert (lens == 50).all() and (ids[:, 50:] == INVALID).all() and np.isinf(dist[:, 50:]).all()


def test_empty_and_one_point_index(abi, oracle):
    q = datagen.uniform(3, 8, 11)
    ids, dist, lens = flat(abi, np.zeros((0, 8), np.float32)).exact_search(q, 4)
    assert (ids == INVALID).all() and np.isinf(dist).all() and (lens == 0).all()
    check_l2(abi, oracle, datagen.uniform(1, 8, 12), q, 4)


@pytest.mark.parametrize("nq", [1, 33, 1000])
def test_query_counts(abi, oracle, nq):
    check_l2(abi, oracle, datagen.uniform(4000, 64, 13), datagen.uniform(nq, 64, 14), 10)


def test_batch_larger_than_one_scratch_chunk(abi, oracle, monkeypatch):
    monkeypatch.setenv("IDB_EXACT_SCRATCH_KEYS", "3000")  # read when the index is created: chunks of a few queries
    check_l2(abi, oracle, datagen.uniform(5000, 32, 15), datagen.uniform(301, 32, 16), 10)
    check_l2(abi, oracle, datagen.uniform(5000, 32, 15), datagen.uniform(77, 32, 16), 100)


def test_many_ragged_slices(abi, oracle):
    pts = datagen.uniform(20011, 48, 17)  # a few queries: 20 slices of 1001 rows, the last one 992
    check_l2(abi, oracle, pts, datagen.uniform(5, 48, 18), 10)
    check_l2(abi, oracle, pts, datagen.uniform(5, 48, 18), 100)


def test_exact_ties_across_slices(abi, oracle):
    pts = datagen.grid_ties(20011, 3, 19, side=4)  # integer grid: many equal distances
    dup = pts[5].copy()
    for b in (0, 1000, 1001, 1002, 5004, 10009, 20010):  # the same row at and around slice boundaries
        pts[b] = dup
    q = np.concatenate([dup[None, :], datagen.grid_ties(20, 3, 20, side=4)]).astype(np.float32)
    ix = check_l2(abi, oracle, pts, q, 10)
    ids, dist, _ = ix.exact_search(q[:1], 10)
    assert ids[0, 0] == 0 and dist[0, 0] == 0.0  # equal keys: the lowest PointId first


def test_special_values(abi, oracle):
    rng = np.random.default_rng(21)
    pts = rng.random((1000, 20), dtype=np.float32)
    pts[10] = 1e-39   # subnormal elements
    pts[11] = 1e20    # the squared distance overflows to +inf
    pts[12, 3] = np.nan  # a row with NaN: NaN distance to every query, ordered last
    pts[13] = 0.0
    q = rng.random((6, 20), dtype=np.float32)
    q[0] = pts[100]   # distance 0
    q[1] = 0.0
    q[2] = 2e-39
    q[3, 5] = np.nan  # a query with NaN: every distance NaN, ties by PointId
    check_l2(abi, oracle, pts, q, 1000)  # the whole order, NaN row last
    # cosine: a NaN query element makes every distance NaN, written as 0x7fc00000
    ix = flat(abi, abi.normalize(pts[:10]), metric="cosine")
    ids, dist, lens = ix.exact_search(q[3:4], 10)
    assert (dist.view(np.uint32) == 0x7FC00000).all() and (ids == np.arange(10)).all() and lens[0] == 10


@pytest.mark.parametrize("n", [1000, 5000])  # one slice (the scan writes the results) / several (K4, then the id map)
def test_adopted_loaded_and_built_agree_and_map_ids(abi, oracle, tmp_path, n):
    pts = datagen.sift_shaped(n, 40, 22)
    q = datagen.sift_shaped(50, 40, 23)
    built, _ = abi.Index.build(pts, seed=3)
    stored, zero, upper = built.export_graph()
    adopted = abi.Index.from_graph(stored, zero, upper, 32)
    path = str(tmp_path / "g.idx")
    built.save(path)
    loaded, _ = abi.Index.load(path, dim=40, M=32)
    want_ids, want_dist = oracle.bruteforce(stored, q, 10)
    gmap = np.random.default_rng(24).permutation(n).astype(np.uint32) + 1000
    for ix in (built, adopted, loaded):
        assert_same(ix.exact_search(q, 10), want_ids, want_dist)
        ix.set_id_map(gmap)
        ids, dist, lens = ix.exact_search(q, 10)
        assert (ids == gmap[want_ids]).all() and dist.tobytes() == want_dist.tobytes() and (lens == 10).all()


def test_device_entry_unaligned_unpadded_on_every_lane(abi, oracle):
    import torch

    n, dim, nq, k = 3000, 30, 45, 16
    pts = datagen.uniform(n, dim, 25)
    q = datagen.uniform(nq, dim, 26)
    ix = flat(abi, pts)
    want_ids, want_dist = oracle.bruteforce(pts, q, k)
    buf = torch.zeros(nq * dim + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(q.ravel()).cuda()  # 4-byte aligned rows of 30 floats
    torch.cuda.synchronize()
    for lane in range(abi.lib().idb_index_num_lanes()):
        ids = torch.empty(nq * k, dtype=torch.int32, device="cuda")
        dist = torch.empty(nq * k, dtype=torch.float32, device="cuda")
        lens = torch.empty(nq, dtype=torch.int32, device="cuda")
        ix.exact_search_device(buf.data_ptr() + 4, nq, k, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=lane)
        ix.sync()
        got = (ids.cpu().numpy().view(np.uint32).reshape(nq, k), dist.cpu().numpy().reshape(nq, k), lens.cpu().numpy().view(np.uint32))
        assert_same(got, want_ids, want_dist)


def test_exact_and_approximate_searches_at_once(abi, oracle):
    pts = datagen.sift_shaped(6000, 64, 27)
    q = datagen.sift_shaped(400, 64, 28)
    ix, _ = abi.Index.build(pts, seed=5)
    want_exact = ix.exact_search(q, 10)
    want_approx = ix.search(q, ef_search=64, k=10)
    bad = []

    def run(fn, want):
        for _ in range(5):
            got = fn()
            if not all(np.array_equal(a, b) for a, b in zip(got, want)):
                bad.append(fn)

    ts = [threading.Thread(target=run, args=(lambda: ix.exact_search(q, 10), want_exact)),
          threading.Thread(target=run, args=(lambda: ix.search(q, ef_search=64, k=10), want_approx))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not bad


def test_one_million_rows(abi, oracle):
    pts = datagen.sift_shaped(1_000_000, 128, 29)
    q = datagen.sift_shaped(1000, 128, 30)
    check_l2(abi, oracle, pts, q, 10)
