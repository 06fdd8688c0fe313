"""The cosine metric on the GPU (DESIGN.md §3a), compared bit for bit with its CPU statement (tests/cosine_ref.py: the oracle's
canonical squared L2 on canonically normalised rows, distances halved): the canonical normalisation,
search on an adopted cosine graph (ids, distance bytes, lengths, per-layer counters), the build, save / load, the sharded path and
the Python module."""
import numpy as np
import pytest

from tests import cosine_ref as cref
from tests import datagen

pytestmark = pytest.mark.gpu


def bf16_round(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u.astype(np.uint64) + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _same(got, want):
    assert (got[2] == want[2]).all()
    assert (got[0] == want[0]).all(), f"{(got[0] != want[0]).any(axis=1).sum()} of {len(got[0])} queries differ"
    assert got[1].tobytes() == want[1].tobytes()


def _cosine_graph(oracle, pts, seed, M=32, threads=4):
    ix, ids = cref.build(oracle, pts, seed=seed, M=M, threads=threads)
    return ix, ix.export(), ids


@pytest.mark.parametrize("dim", [1, 3, 30, 128, 300, 768, 1100, 4100])
def test_normalize_equals_oracle(abi, oracle, dim):
    rng = np.random.default_rng(dim)
    x = (rng.standard_normal((40, dim)) * rng.choice([1e-20, 1e-3, 1.0, 1e4], (40, 1))).astype(np.float32)
    x[1] = 0.0
    x[2, 0] = np.nan
    x[3] = 1e20  # the sum of squares overflows: zeros
    x[4, -1] = np.inf  # inf / inf: NaN
    got, want = abi.normalize(x), cref.normalize(oracle, x)
    assert got.tobytes() == want.tobytes()
    assert (got[1] == 0).all() and (got[3] == 0).all() and np.isnan(got[2]).all()


@pytest.mark.parametrize("n,dim,M,ef", [(3000, 128, 32, 100), (4000, 30, 16, 64), (2000, 300, 24, 128), (3000, 5, 32, 200),
                                        (1000, 1536, 32, 64), (600, 4100, 16, 50)])
def test_search_parity_on_an_oracle_cosine_graph(abi, oracle, n, dim, M, ef):
    pts = datagen.uniform(n, dim, 300 + dim) * 2 - 1
    ix_o, g, _ = _cosine_graph(oracle, pts, seed=n, M=M)
    q = datagen.uniform(200, dim, 301 + dim) * 2 - 1
    q[7] = 0.0  # a zero query stays zero: 0.5 from every point
    gpu = abi.Index.from_graph(g.points, g.zero, g.upper, g.M, metric="cosine")
    assert gpu.metric == "cosine"
    got = gpu.search(q, ef_search=ef, k=ef)
    want = cref.search(oracle, ix_o, q, ef_search=ef, k=ef, counters=True)
    _same(got, want)
    assert (gpu.last_counters(len(q)) == want[3]).all()
    fin = got[1][~np.isnan(got[1])]
    assert (fin >= 0).all() and (fin <= 2.0).all()
    gpu.close()


FLAVOURS = {"b16": {}, "bitmap": {"IDB_VIS_TIER": "1"}, "hash": {"IDB_VIS_TIER": "0"}}


@pytest.mark.parametrize("flavour", sorted(FLAVOURS))
def test_every_visited_flavour_and_bf16(abi, oracle, monkeypatch, flavour):
    for k_, v_ in FLAVOURS[flavour].items():
        monkeypatch.setenv(k_, v_)
    pts = datagen.sift_shaped(5000, 128, 11)
    ix_o, g, _ = _cosine_graph(oracle, pts, seed=5)
    q = datagen.sift_shaped(300, 128, 12)
    gpu = abi.Index.from_graph(g.points, g.zero, g.upper, g.M, metric="cosine")
    _same(gpu.search(q, ef_search=100, k=10), cref.search(oracle, ix_o, q, ef_search=100, k=10))
    gpu.close()
    # bf16 storage: the oracle on the bf16-rounded unit rows (which the from_graph check lets through)
    rp = bf16_round(g.points)
    ox = oracle.from_graph(oracle.Graph(rp, g.zero, g.upper, g.M, 100))
    gb = abi.Index.from_graph(g.points, g.zero, g.upper, g.M, storage="bf16", metric="cosine")
    got, want = gb.search(q, ef_search=100, k=10), cref.search(oracle, ox, q, ef_search=100, k=10, counters=True)
    _same(got, want)
    assert (gb.last_counters(len(q)) == want[3]).all()
    gb.close()


def test_retry_pass_reads_the_same_normalised_queries(abi, oracle, monkeypatch):
    """Queries overflowing a 1024-slot visited table are re-run by the retry pass; it must see the rows K1 saw (normalised once)."""
    pts = datagen.uniform(20_000, 16, 13) * 2 - 1
    ix_o, g, _ = _cosine_graph(oracle, pts, seed=3, threads=8)
    q = datagen.uniform(300, 16, 14) * 2 - 1
    want = cref.search(oracle, ix_o, q, ef_search=100, k=10, counters=True)
    assert want[3][:, 3].max() > 1000
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    gpu = abi.Index.from_graph(g.points, g.zero, g.upper, g.M, metric="cosine")
    q_before = q.copy()
    _same(gpu.search(q, ef_search=100, k=10), want)
    assert gpu.last_retried(0xFFFFFFFF) > 0
    assert (gpu.last_counters(len(q)) == want[3]).all()
    assert q.tobytes() == q_before.tobytes()
    gpu.set_profiling(True)  # one more launch than an L2 call: the normalisation
    gpu.search(q[:10], ef_search=100, k=10)
    assert gpu.last_kernel_ms()[1] == 3
    gpu.close()


def test_device_api_does_not_write_the_callers_queries(abi, oracle):
    import torch

    pts = datagen.uniform(3000, 30, 21) * 2 - 1
    ix_o, g, _ = _cosine_graph(oracle, pts, seed=2)
    q = datagen.uniform(500, 30, 22) * 2 - 1
    gpu = abi.Index.from_graph(g.points, g.zero, g.upper, g.M, metric="cosine")
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((500, 10), dtype=torch.int32, device="cuda")
    dist = torch.empty((500, 10), dtype=torch.float32, device="cuda")
    lens = torch.empty((500,), dtype=torch.int32, device="cuda")
    gpu.search_device(dq.data_ptr(), 500, 60, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=1)
    torch.cuda.synchronize()
    want = cref.search(oracle, ix_o, q, ef_search=60, k=10)
    _same((ids.cpu().numpy().view(np.uint32), dist.cpu().numpy(), lens.cpu().numpy().view(np.uint32)), want)
    assert dq.cpu().numpy().tobytes() == q.tobytes()
    gpu.close()


@pytest.mark.parametrize("storage,dim", [("f32", 64), ("bf16", 128), ("f32", 1100)])
def test_sequential_build_equals_oracle_build(abi, oracle, storage, dim):
    pts = datagen.sift_shaped(1500, dim, 8)
    ix_o, g, ids_o = _cosine_graph(oracle, pts, seed=12, threads=1)
    if storage == "bf16":  # normalised in f32, then rounded: the traversal is the canonical squared L2 on those rows
        ix_o, ids_o = oracle.build(bf16_round(cref.normalize(oracle, pts)), seed=12, threads=1)
        g = ix_o.export()
    ix_g, ids_g = abi.Index.build(pts, seed=12, insert_batch=1, storage=storage, metric="cosine")
    p, zero, upper = ix_g.export_graph()
    assert (ids_g == ids_o).all() and p.tobytes() == g.points.tobytes() and (zero == g.zero).all()
    assert all((a == b).all() for a, b in zip(upper, g.upper))
    ix_g.close()


def test_batched_build_recall(abi, oracle):
    pts = datagen.sift_shaped(20000, 128, 3)
    q = datagen.sift_shaped(300, 128, 4)
    ix, ids = abi.Index.build(pts, seed=2, metric="cosine")
    inv = np.empty(len(ids), np.int64)
    inv[ids] = np.arange(len(ids))
    truth, _ = cref.bruteforce(oracle, pts, q, 10, threads=8)
    got, _, _ = ix.search(q, ef_search=100, k=10)
    rec = np.mean([len(set(inv[a].tolist()) & set(b.tolist())) / 10 for a, b in zip(got, truth)])
    assert rec > 0.95, rec
    ix.close()


def test_save_load_round_trip(abi, oracle, tmp_path):
    pts = datagen.sift_shaped(4000, 40, 5)
    q = datagen.sift_shaped(200, 40, 6)
    ix, _ = abi.Index.build(pts, seed=4, metric="cosine")
    before = ix.search(q, ef_search=80, k=20)
    path = str(tmp_path / "cos.idx")
    ix.save(path)
    back, _ = abi.Index.load(path, dim=40, M=32, metric="cosine")
    assert back.metric == "cosine"
    _same(back.search(q, ef_search=80, k=20), before)
    l2, _ = abi.Index.load(path, dim=40, M=32)  # the same file as a squared-L2 index, searched with the normalised queries:
    got = l2.search(abi.normalize(q), ef_search=80, k=20)  # the same traversal, the key distances (twice the reported ones)
    assert (got[0] == before[0]).all() and (got[1] == 2 * before[1]).all()
    [x.close() for x in (ix, back, l2)]


def test_from_graph_ex_rejects_non_unit_rows(abi, oracle):
    pts = datagen.uniform(500, 16, 9)
    ix_o, g, _ = _cosine_graph(oracle, pts, seed=1)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(pts, g.zero, g.upper, g.M, metric="cosine")  # the raw rows: not unit length
    assert e.value.status == abi.ERR_INVALID_ARG
    bad = g.points.copy()
    bad[123] *= 1.02
    with pytest.raises(abi.IdbError):
        abi.Index.from_graph(bad, g.zero, g.upper, g.M, metric="cosine")
    ok = g.points.copy()
    ok[5] = 0.0  # all-zero rows are accepted
    abi.Index.from_graph(ok, g.zero, g.upper, g.M, metric="cosine").close()


def test_sharded_world_of_one_equals_the_host_protocol(abi, oracle):
    from instant_distance_b200 import sharded

    n_sh, per, dim, k, ef = 2, 4000, 48, 10, 100
    q = datagen.sift_shaped(600, dim, 31)
    shards, keys = [], []
    for s in range(n_sh):
        ix, ids = abi.Index.build(datagen.sift_shaped(per, dim, 40 + s), seed=50 + s, metric="cosine")
        gmap = sharded.global_id_map(ids, s * per)
        p, zero, upper = ix.export_graph()
        ox = oracle.from_graph(oracle.Graph(p, zero, upper, 32, ef))
        o_ids, o_dist, o_len = cref.search(oracle, ox, q, ef_search=ef, k=k, threads=8)
        _same(ix.search(q, ef_search=ef, k=k), (o_ids, o_dist, o_len))
        gids = np.where(o_ids == 0xFFFFFFFF, 0, gmap[np.minimum(o_ids, per - 1)])
        keys.append(sharded.pack_keys(o_dist, gids, np.minimum(o_len, k)))  # (1 - cos orders as the traversal keys do)
        ix.set_id_map(gmap)
        shards.append(ix)
    comm = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    got = abi.sharded_search_multi(shards, comm, q, ef_search=ef, k=k)
    _same(got, sharded.merge_keys(np.stack(keys), k))
    # mixed metrics in one call are rejected
    l2, _ = abi.Index.build(datagen.sift_shaped(per, dim, 49), seed=59)
    with pytest.raises(abi.IdbError) as e:
        abi.sharded_search_multi([shards[0], l2], comm, q, ef_search=ef, k=k)
    assert e.value.status == abi.ERR_INVALID_ARG
    comm.close()
    [s_.close() for s_ in shards + [l2]]


def test_python_module_cosine(abi, oracle, tmp_path):
    import instant_distance as idist

    pts = datagen.sift_shaped(3000, 24, 61)
    cfg = idist.Config()
    cfg.seed, cfg.metric = 7, "cosine"
    hnsw, ids = idist.Hnsw.build([list(p) for p in pts], cfg)
    q = pts[10] * 3.0  # same direction: distance 0 (up to rounding) to point 10
    s = idist.Search()
    hnsw.search(list(q), s)
    first = next(iter(s))
    assert ids[10] == first.pid and abs(first.distance) < 1e-6
    ids_many, dist_many, _ = hnsw.search_many(pts[:50], k=5)
    path = str(tmp_path / "h.idx")
    hnsw.dump(path)
    back = idist.Hnsw.load(path, dim=24, M=32, metric="cosine")
    ids2, dist2, _ = back.search_many(pts[:50], k=5)
    assert (ids2 == ids_many).all() and dist2.tobytes() == dist_many.tobytes()
    vals = [f"v{i}" for i in range(len(pts))]
    m = idist.HnswMap.build([list(p) for p in pts], vals, cfg)
    m.dump(path)
    mb = idist.HnswMap.load(path, dim=24, M=32, metric="cosine")
    s2 = idist.Search()
    mb.search(list(pts[3]), s2)
    assert next(iter(s2)).value == "v3"
