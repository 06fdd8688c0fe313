"""The search entry points of each family give byte-identical ids, distances and lengths whichever way the queries and results
travel: host buffers (pageable or pinned, with or without distances and lengths) and device buffers (16-byte aligned or not, on lane
0 or another lane).  Each result also equals the CPU statement: the oracle's search of the same graph (approximate and sharded
entries, with the per-layer counters) or oracle.bruteforce over the stored rows (exact entries).  Also pinned: the caller's queries
are never written, the launch count idb_index_last_kernel_ms reports, and which lane's diagnostics a call leaves behind."""
import ctypes as C

import numpy as np
import pytest

from tests import cosine_ref, datagen
from tests import merge_statement as ms
from tests.test_gpu_sharded import THREADS, Spec, _check_fused, _oracle_keys, _shards

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF
NQ = 40


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


@pytest.fixture(scope="module")
def comm(abi):
    c = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    yield c
    c.close()


class HostOut:
    """Host result buffers: pageable numpy arrays, or numpy views of idb_host_alloc'd (pinned) memory.  `full=False`: no distances
    and no lengths."""

    def __init__(self, abi, nq, k, pinned, full=True):
        self.abi, self.ptrs = abi, []
        self.ids = self._arr(nq * k, np.uint32, pinned).reshape(nq, k)
        self.dist = self._arr(nq * k, np.float32, pinned).reshape(nq, k) if full else None
        self.lens = self._arr(nq, np.uint32, pinned) if full else None

    def _arr(self, n, dt, pinned):
        if not pinned:
            return np.full(n, 0xAB, dtype=dt)
        p = C.c_void_p()
        self.abi.check(self.abi.lib().idb_host_alloc(max(4, n * 4), C.byref(p)))
        self.ptrs.append(p)
        a = np.ctypeslib.as_array((C.c_uint32 * max(1, n)).from_address(p.value))[:n].view(dt)
        a.view(np.uint32)[:] = 0xABABABAB
        return a

    def args(self):
        def p(a, t):
            return None if a is None else a.ctypes.data_as(C.POINTER(t))
        return p(self.ids, C.c_uint32), p(self.dist, C.c_float), p(self.lens, C.c_uint32)

    def result(self):
        out = (self.ids.copy(), None if self.dist is None else self.dist.copy(), None if self.lens is None else self.lens.copy())
        for p in self.ptrs:
            self.abi.lib().idb_host_free(p)
        self.ptrs = []
        return out


class DevQueries:
    """The queries on the device, at a 16-byte-aligned address or one float past it."""

    def __init__(self, q, aligned):
        import torch

        self.buf = torch.zeros(q.size + 4, dtype=torch.float32, device="cuda")
        self.off = 0 if aligned else 1
        self.buf[self.off:self.off + q.size] = torch.from_numpy(np.ascontiguousarray(q).ravel()).cuda()
        self.ptr = self.buf.data_ptr() + 4 * self.off
        self.before = self.buf.cpu().numpy().tobytes()

    def unchanged(self):
        import torch

        torch.cuda.synchronize()
        return self.buf.cpu().numpy().tobytes() == self.before


class DevOut:
    def __init__(self, nq, k, full=True):
        import torch

        self.ids = torch.full((max(1, nq * k),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        self.dist = torch.full((max(1, nq * k),), 0x5A5A5A5A, dtype=torch.int32, device="cuda") if full else None
        self.lens = torch.full((max(1, nq),), 0x5A5A5A5A, dtype=torch.int32, device="cuda") if full else None
        self.nq, self.k = nq, k

    def args(self):
        return tuple(None if t is None else t.data_ptr() for t in (self.ids, self.dist, self.lens))

    def result(self):
        import torch

        torch.cuda.synchronize()
        nq, k = self.nq, self.k
        ids = self.ids.cpu().numpy().view(np.uint32)[:nq * k].reshape(nq, k)
        dist = None if self.dist is None else self.dist.cpu().numpy().view(np.float32)[:nq * k].reshape(nq, k)
        lens = None if self.lens is None else self.lens.cpu().numpy().view(np.uint32)[:nq]
        return ids, dist, lens


def _eq(got, want, what):
    """Byte equality of (ids, dist, lens); a None part of `got` is not compared."""
    assert (got[0] == want[0]).all(), f"{what}: ids differ in {(got[0] != want[0]).any(axis=1).sum()} of {len(got[0])} queries"
    if got[1] is not None:
        assert got[1].tobytes() == want[1].tobytes(), f"{what}: distance bytes differ"
    if got[2] is not None:
        assert (got[2] == want[2]).all(), f"{what}: lengths differ"


# ==== the approximate and exact families ======================================================================================

def _approx_host(abi, ix, q, ef, k, pinned=False, full=True):
    ho = HostOut(abi, len(q), k, pinned, full)
    abi.check(abi.lib().idb_search_batch_f32(ix._h, q.ctypes.data_as(C.POINTER(C.c_float)), len(q), ef, k, *ho.args()))
    return ho.result()


def _approx_device(abi, ix, q, ef, k, aligned=True, lane=None, full=True):
    dq, do = DevQueries(q, aligned), DevOut(len(q), k, full)
    if lane is None:
        abi.check(abi.lib().idb_search_batch_device(ix._h, dq.ptr, len(q), ef, k, *do.args()))
    else:
        abi.check(abi.lib().idb_search_batch_device_lane(ix._h, lane, dq.ptr, len(q), ef, k, *do.args()))
    ix.sync()
    assert dq.unchanged(), "the caller's device queries were written"
    return do.result()


def _exact_host(abi, ix, q, k, pinned=False, full=True):
    ho = HostOut(abi, len(q), k, pinned, full)
    abi.check(abi.lib().idb_exact_search_batch_f32(ix._h, q.ctypes.data_as(C.POINTER(C.c_float)), len(q), k, *ho.args()))
    return ho.result()


def _exact_device(abi, ix, q, k, aligned=True, lane=0, full=True):
    dq, do = DevQueries(q, aligned), DevOut(len(q), k, full)
    abi.check(abi.lib().idb_exact_search_batch_device_lane(ix._h, lane, dq.ptr, len(q), k, *do.args()))
    ix.sync()
    assert dq.unchanged(), "the caller's device queries were written"
    return do.result()


def _approx_want(oracle, sh, q, ef, k):
    """The oracle's search through the id map: (ids, dist, lens = len(nearest), which may exceed k), and its counters."""
    keys, cnt = _oracle_keys(oracle, sh, q, ef, k)
    ids, dist, _ = ms.merge(keys[None], k, sh.spec.metric)
    qq = cosine_ref.normalize(oracle, q) if sh.spec.metric == "cosine" else q
    lens = sh.ox.search(qq, ef_search=min(ef, sh.spec.n), k=k, counters=True, threads=THREADS)[2]
    return (ids, dist, np.asarray(lens, dtype=np.uint32)), cnt


def _exact_want(abi, oracle, sh, q, k):
    rows = sh.ix.export_graph()[0]
    qq = cosine_ref.normalize(oracle, q) if sh.spec.metric == "cosine" else q
    ids, dist = oracle.bruteforce(rows, qq, k, threads=THREADS)
    if sh.spec.metric == "cosine":
        dist = cosine_ref.reported(dist)
    real = ids != INVALID
    ids = np.where(real, sh.gmap[np.where(real, ids, 0)], INVALID).astype(np.uint32)
    return ids, np.ascontiguousarray(dist, dtype=np.float32), real.sum(1).astype(np.uint32)


CASES = [(d, st, m) for d in (48, 45, 1030) for st in ("f32", "bf16") for m in ("l2sq", "cosine")]


@pytest.mark.parametrize("dim,storage,metric", CASES, ids=[f"dim{d}-{st}-{m}" for d, st, m in CASES])
def test_every_way_in_and_out_gives_the_same_bytes(abi, oracle, dim, storage, metric):
    (sh,) = _shards(abi, oracle, [Spec(1500, dim, storage, metric, M=16, ef=64)])
    ix, ef, k = sh.ix, 64, 20
    q = datagen.sift_shaped(NQ, dim, 900 + dim) - (60.0 if metric == "cosine" else 0.0)
    q_before = q.tobytes()

    want, cnt = _approx_want(oracle, sh, q, ef, k)
    _eq(_approx_host(abi, ix, q, ef, k), want, "approximate host, pageable")
    assert (ix.last_counters(NQ) == cnt).all(), "approximate host: per-layer counters"
    _eq(_approx_host(abi, ix, q, ef, k, pinned=True), want, "approximate host, pinned")
    _eq(_approx_host(abi, ix, q, ef, k, full=False), want, "approximate host, ids only")
    for aligned in (True, False):
        _eq(_approx_device(abi, ix, q, ef, k, aligned), want, f"approximate device, aligned={aligned}")
        assert (ix.last_counters(NQ) == cnt).all(), "approximate device: per-layer counters"
        _eq(_approx_device(abi, ix, q, ef, k, aligned, lane=3), want, f"approximate device lane 3, aligned={aligned}")
        assert (ix.last_counters(NQ) == cnt).all(), "approximate device lane 3: per-layer counters"
    _eq(_approx_device(abi, ix, q, ef, k, lane=2, full=False), want, "approximate device, ids only")

    want = _exact_want(abi, oracle, sh, q, k)
    _eq(_exact_host(abi, ix, q, k), want, "exact host, pageable")
    _eq(_exact_host(abi, ix, q, k, pinned=True), want, "exact host, pinned")
    _eq(_exact_host(abi, ix, q, k, full=False), want, "exact host, ids only")
    for aligned in (True, False):
        for lane in (0, 2):
            _eq(_exact_device(abi, ix, q, k, aligned, lane), want, f"exact device lane {lane}, aligned={aligned}")
    _eq(_exact_device(abi, ix, q, k, lane=1, full=False), want, "exact device, ids only")
    assert q.tobytes() == q_before, "the caller's host queries were written"


@pytest.mark.parametrize("storage", ["f32", "bf16"])
def test_k_above_n(abi, oracle, storage):
    (sh,) = _shards(abi, oracle, [Spec(30, 45, storage, ef=100)])
    q = datagen.sift_shaped(NQ, 45, 5)
    want, _ = _approx_want(oracle, sh, q, 100, 64)
    assert (want[2] == 30).all()
    for got in (_approx_host(abi, sh.ix, q, 100, 64), _approx_device(abi, sh.ix, q, 100, 64, aligned=False),
                _approx_device(abi, sh.ix, q, 100, 64, lane=1)):
        _eq(got, want, "approximate, k > n")
    want = _exact_want(abi, oracle, sh, q, 64)
    for got in (_exact_host(abi, sh.ix, q, 64), _exact_device(abi, sh.ix, q, 64, aligned=False)):
        _eq(got, want, "exact, k > n")


def _empty_lists(nq, k):
    return (np.full((nq, k), INVALID, np.uint32), np.full((nq, k), np.inf, np.float32), np.zeros(nq, np.uint32))


@pytest.mark.parametrize("case", ["empty-index", "ef0"])
def test_empty_results(abi, case):
    """An empty index, and ef_search = 0 in the call on an index whose own default is 0: empty result lists."""
    n = 0 if case == "empty-index" else 8
    pts = datagen.uniform(n, 45, 1).astype(np.float32).reshape(n, 45)
    ix = abi.Index.from_graph(pts, np.full((n, 32), INVALID, np.uint32), [], 16, ef_search=0 if case == "ef0" else 50)
    q, k, ef = datagen.uniform(NQ, 45, 2), 10, 0
    want = _empty_lists(NQ, k)
    for pinned in (False, True):
        _eq(_approx_host(abi, ix, q, ef, k, pinned=pinned), want, f"approximate host, pinned={pinned}")
    for aligned in (True, False):
        _eq(_approx_device(abi, ix, q, ef, k, aligned), want, f"approximate device, aligned={aligned}")
        _eq(_approx_device(abi, ix, q, ef, k, aligned, lane=2), want, f"approximate device lane 2, aligned={aligned}")
    if n == 0:
        for got in (_exact_host(abi, ix, q, k), _exact_host(abi, ix, q, k, pinned=True), _exact_device(abi, ix, q, k, aligned=False),
                    _exact_device(abi, ix, q, k, lane=3)):
            _eq(got, want, "exact, empty index")
    ix.close()


def test_no_queries_writes_nothing(abi, oracle, comm):
    (sh,) = _shards(abi, oracle, [Spec(300, 45)])
    L, h = abi.lib(), sh.ix._h
    ho = HostOut(abi, 1, 8, pinned=False)
    do = DevOut(1, 8)
    q = np.zeros((1, 45), np.float32)
    qp = q.ctypes.data_as(C.POINTER(C.c_float))
    one = (C.c_void_p * 1)(h)
    for st in (L.idb_search_batch_f32(h, qp, 0, 0, 8, *ho.args()), L.idb_search_batch_device(h, q.ctypes.data, 0, 0, 8, *do.args()),
               L.idb_search_batch_device_lane(h, 1, q.ctypes.data, 0, 0, 8, *do.args()),
               L.idb_exact_search_batch_f32(h, qp, 0, 8, *ho.args()),
               L.idb_exact_search_batch_device_lane(h, 1, q.ctypes.data, 0, 8, *do.args()),
               L.idb_sharded_search_batch_f32(h, comm._h, qp, 0, 0, 8, *ho.args()),
               L.idb_sharded_search_batch_device(h, comm._h, q.ctypes.data, 0, 0, 8, *do.args()),
               L.idb_sharded_search_batch_f32_multi(one, 1, comm._h, qp, 0, 0, 8, *ho.args()),
               L.idb_sharded_search_batch_device_multi(one, 1, comm._h, q.ctypes.data, 0, 0, 8, *do.args())):
        assert st == abi.OK
    sh.ix.sync()
    assert (ho.ids == 0xAB).all() and (ho.lens == 0xAB).all()
    assert (do.result()[0] == 0x5A5A5A5A).all()


@pytest.mark.parametrize("metric", ["l2sq", "cosine"])
def test_launch_count_and_lane_diagnostics(abi, oracle, metric):
    (sh,) = _shards(abi, oracle, [Spec(1500, 45, metric=metric)])
    ix = sh.ix
    q = datagen.sift_shaped(NQ, 45, 7)
    ix.set_profiling(True)
    want_launches = 3 if metric == "cosine" else 2
    _approx_device(abi, ix, q, 64, 10, lane=2)
    assert ix.last_kernel_ms()[1] == want_launches
    cell = ix.last_kernel()  # the latest call's lane
    assert cell == ix.last_kernel(2) and any(cell.values())
    assert not any(ix.last_kernel(1).values())
    # exact calls leave the lane diagnostics alone
    _exact_device(abi, ix, q, 10, lane=1)
    _exact_host(abi, ix, q, 10)
    assert ix.last_kernel() == cell and not any(ix.last_kernel(1).values())
    assert ix.last_kernel_ms()[1] == want_launches
    # a host call takes a lane and makes it the latest
    _approx_host(abi, ix, q, 64, 10)
    assert ix.last_kernel_ms()[1] == want_launches and ix.last_kernel() == cell
    ix.set_profiling(False)


# ==== the sharded family ======================================================================================================

def _sharded_host(abi, shards, comm, q, ef, k, multi, pinned=False, full=True):
    ho = HostOut(abi, len(q), k, pinned, full)
    qp = q.ctypes.data_as(C.POINTER(C.c_float))
    L = abi.lib()
    if multi:
        hs = (C.c_void_p * len(shards))(*[s.ix._h for s in shards])
        abi.check(L.idb_sharded_search_batch_f32_multi(hs, len(shards), comm._h, qp, len(q), ef, k, *ho.args()))
    else:
        abi.check(L.idb_sharded_search_batch_f32(shards[0].ix._h, comm._h, qp, len(q), ef, k, *ho.args()))
    return ho.result()


def _sharded_device(abi, shards, comm, q, ef, k, multi, aligned=True, full=True):
    dq, do = DevQueries(q, aligned), DevOut(len(q), k, full)
    L = abi.lib()
    if multi:
        hs = (C.c_void_p * len(shards))(*[s.ix._h for s in shards])
        abi.check(L.idb_sharded_search_batch_device_multi(hs, len(shards), comm._h, dq.ptr, len(q), ef, k, *do.args()))
    else:
        abi.check(L.idb_sharded_search_batch_device(shards[0].ix._h, comm._h, dq.ptr, len(q), ef, k, *do.args()))
    for s in shards:
        s.ix.sync()
    assert dq.unchanged(), "the caller's device queries were written"
    return do.result()


SHARD_CASES = [(d, st, m) for d in (48, 45, 1030) for st, m in (("f32", "l2sq"), ("bf16", "l2sq"), ("f32", "cosine"))]


@pytest.mark.parametrize("dim,storage,metric", SHARD_CASES, ids=[f"dim{d}-{st}-{m}" for d, st, m in SHARD_CASES])
def test_sharded_every_way_in_and_out(abi, oracle, comm, dim, storage, metric):
    shards = _shards(abi, oracle, [Spec(1200, dim, storage, metric)] * 3)
    q = datagen.sift_shaped(NQ, dim, 77) - (60.0 if metric == "cosine" else 0.0)
    q_before = q.tobytes()
    ef, k = 64, 20
    shards[0].ix.set_profiling(True)
    got = _sharded_host(abi, shards, comm, q, ef, k, multi=True)
    _check_fused(oracle, shards, got, q, ef, k, "sharded host")  # every shard's K1 cell and counters, the merged lists
    per = 3 if metric == "cosine" else 2
    assert shards[0].ix.last_kernel_ms()[1] == per * 3 + 1 + 2
    for variant in ({"pinned": True}, {"full": False}):
        _eq(_sharded_host(abi, shards, comm, q, ef, k, multi=True, **variant), got, f"sharded host {variant}")
    for aligned in (True, False):
        dev = _sharded_device(abi, shards, comm, q, ef, k, multi=True, aligned=aligned)
        _check_fused(oracle, shards, dev, q, ef, k, f"sharded device, aligned={aligned}")
        _eq(dev, got, f"sharded device, aligned={aligned}")
    _eq(_sharded_device(abi, shards, comm, q, ef, k, multi=True, full=False), got, "sharded device, ids only")
    assert q.tobytes() == q_before, "the caller's host queries were written"

    one = shards[:1]
    got1 = _sharded_host(abi, one, comm, q, ef, k, multi=False)
    _check_fused(oracle, one, got1, q, ef, k, "one shard, host")
    assert shards[0].ix.last_kernel_ms()[1] == per + 2
    _eq(_sharded_device(abi, one, comm, q, ef, k, multi=False, aligned=False), got1, "one shard, device")
    for s in shards:  # a sharded call runs on lane 0 of every shard
        assert s.ix.last_kernel() == s.ix.last_kernel(0)
    shards[0].ix.set_profiling(False)


def test_sharded_empty_and_k_above_n(abi, oracle, comm):
    shards = _shards(abi, oracle, [Spec(0, 45), Spec(30, 45), Spec(1, 45)])
    q = datagen.sift_shaped(NQ, 45, 3)
    got = _sharded_host(abi, shards, comm, q, 0, 64, multi=True)
    _check_fused(oracle, shards, got, q, 0, 64, "empty, small and one-point shards")
    _eq(_sharded_device(abi, shards, comm, q, 0, 64, multi=True, aligned=False), got, "device")
    assert (got[2] == 31).all()
