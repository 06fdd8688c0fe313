"""The sharded search on one GPU, bit for bit against plain statements.

Two parts:
  * K4, the merge kernel (`merge_topk_kernel`, csrc/sharded.cu), alone: `Index.merge_topk` runs it through the same launch as the
    product (`launch_merge`: warps per block, the > 48 KB shared-memory attribute, the grid cap) on key sets built to be hard, and
    its ids, distance bytes, lengths and keys must equal tests/merge_statement.py.  The widths reach 4, 2 and 1 warps per block,
    the limit of the device's opt-in shared memory and one key past it, and batches that outrun one pass of the capped grid.
  * The fused path end to end (`idb_sharded_search_batch_{f32,device}_multi` with a world-size-1 communicator: per-shard K1 with its
    keys epilogue -> pre-merge -> ncclAllGather -> merge): shards are built on the GPU and adopted by the oracle; the oracle's
    per-shard lists, mapped to global ids, go through the plain merge, and the fused result must equal it.  Every shard must also
    report the K1 cell tests/k1_dispatch.py states and the oracle's per-layer counters.
The real world > 1 path runs in scripts/sharded_check.py, where two GPUs exist.
"""
import functools
import json
import os
import subprocess
import sys
from collections import namedtuple

import numpy as np
import pytest

from tests import cosine_ref, datagen
from tests import merge_statement as ms
from tests.conftest import ROOT
from tests.k1_dispatch import Cell, k1_cell

pytestmark = pytest.mark.gpu

THREADS = min(32, os.cpu_count() or 8)


def _gpu_count():
    from instant_distance_b200 import _abi

    return _abi.lib().idb_device_count()


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


@functools.lru_cache(maxsize=None)
def _device():
    """(opt-in shared memory per block, SM count) of device 0: the merge's limit and its grid cap (num_sms * 8 blocks)."""
    import torch

    p = torch.cuda.get_device_properties(0)
    return int(p.shared_memory_per_block_optin), int(p.multi_processor_count)


@pytest.fixture(scope="module")
def comm(abi):
    c = abi.Comm(abi.comm_unique_id(), 0, 1, 0)
    yield c
    c.close()


# ==== K4 alone ================================================================================================================

@pytest.fixture(scope="module")
def merge_ix(abi):
    """Empty indexes: the merge needs only the device and the metric it reports distances in."""
    out = {m: abi.Index.from_graph(np.zeros((0, 8), np.float32), np.zeros((0, 64), np.uint32), [], 32, metric=m)
           for m in ("l2sq", "cosine")}
    yield out
    [ix.close() for ix in out.values()]


GS = (1, 2, 3, 7, 8, 33, 64)
KS = (1, 2, 31, 32, 33, 100, 1024)
REGIMES = set()  # (warps per block, dynamic shared memory > 48 KB) that a checked merge ran with; "refused" for the refusals
MERGE_DONE = set()  # the merge tests that passed in this session


def _check_merge(merge_ix, keys, k, what):
    want = ms.merged_keys(keys, k)
    for metric, ix in merge_ix.items():
        got = ix.merge_topk(keys, k, premerge=True)
        assert got.tobytes() == want.tobytes(), f"{what}: pre-merge keys differ ({metric} index)"
        ids, dist, lens = ix.merge_topk(keys, k)
        w_ids, w_dist, w_lens = ms.report(want, metric)
        assert (lens == w_lens).all(), f"{what}: lengths differ ({metric})"
        bad = (ids != w_ids).any(axis=1)
        assert not bad.any(), f"{what}: ids differ in {bad.sum()} of {len(ids)} queries (first: {np.argmax(bad)}) ({metric})"
        assert dist.tobytes() == w_dist.tobytes(), f"{what}: distance bytes differ ({metric})"


def _refused(abi, merge_ix, G, k):
    keys = np.full((G, 1, k), ms.KEY_NONE, dtype=np.uint64)
    for ix in merge_ix.values():
        for premerge in (True, False):
            with pytest.raises(abi.IdbError) as e:
                ix.merge_topk(keys, k, premerge=premerge)
            assert e.value.status == abi.ERR_UNSUPPORTED
    REGIMES.add("refused")


def _merge_case(abi, merge_ix, G, k, seed):
    max_smem, _ = _device()
    if not ms.fits(G, k, max_smem):
        _refused(abi, merge_ix, G, k)
        return
    w, per_warp = ms.wpb(G, k, max_smem), G * k * 8
    assert w * per_warp <= max_smem and (w == 4 or 2 * w * per_warp > max_smem), "the most warps (at most 4) whose keys fit"
    for kind in ms.KINDS:  # one query of each kind, then five with every kind
        _check_merge(merge_ix, ms.keyset(kind, G, 1, k, seed), k, f"G {G} k {k} nq 1 {kind}")
    _check_merge(merge_ix, ms.mixed(G, 5, k, seed), k, f"G {G} k {k} nq 5")
    REGIMES.add((w, G * k * 8 * w > 48 * 1024))


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("G", GS)
def test_merge_widths(abi, merge_ix, G, k):
    """Every (G, k) of the grid: the ones whose keys fit run (4, 2 or 1 warps per block), the others are refused."""
    _merge_case(abi, merge_ix, G, k, 100 * G + k)
    MERGE_DONE.add(("widths", G, k))


@pytest.mark.parametrize("G", GS)
def test_merge_at_the_shared_memory_limit(abi, merge_ix, G):
    """The largest k whose G x k keys fit the device's opt-in shared memory per block runs with one warp per block; one more is
    refused."""
    max_smem, _ = _device()
    k = max_smem // (8 * G)
    assert ms.fits(G, k, max_smem) and not ms.fits(G, k + 1, max_smem)
    assert ms.wpb(G, k, max_smem) == 1 and G * k * 8 > 48 * 1024
    _merge_case(abi, merge_ix, G, k, 7 * G)
    _merge_case(abi, merge_ix, G, k + 1, 7 * G)
    MERGE_DONE.add(("limit", G))


def _grid_stride_case(wpb):
    """(G, k) that runs with `wpb` warps per block on this device."""
    max_smem, _ = _device()
    if wpb == 4:
        return 3, 100
    if wpb == 2:
        return 8, 1024
    return 7, max_smem // (8 * 7 * 2) + 1  # just over half the limit per warp


@pytest.mark.parametrize("wpb", (4, 2, 1))
def test_merge_grid_stride_loop(merge_ix, wpb):
    """More queries than one pass of the capped grid (num_sms * 8 blocks of wpb warps, one query per warp) covers: 5 000 at 4
    warps per block, 1.25 times the capped grid's queries at 2 and 1."""
    max_smem, num_sms = _device()
    G, k = _grid_stride_case(wpb)
    assert ms.wpb(G, k, max_smem) == wpb
    cap = num_sms * 8 * wpb
    nq = max(5000, cap + 1) if wpb == 4 else cap * 5 // 4
    assert nq > cap
    _check_merge(merge_ix, ms.mixed(G, nq, k, wpb), k, f"G {G} k {k} nq {nq}")
    REGIMES.add(("grid-stride", wpb))
    MERGE_DONE.add(("grid-stride", wpb))


def test_merge_reached_every_launch_regime():
    wanted = {(4, False), (4, True), (2, True), (1, True), "refused"} | {("grid-stride", w) for w in (4, 2, 1)}
    if len(MERGE_DONE) < len(GS) * len(KS) + len(GS) + 3:
        pytest.skip("needs every merge test of this file in this session")
    assert wanted <= REGIMES, f"never ran: {sorted(map(str, wanted - REGIMES))}"


# ==== the fused path end to end ===============================================================================================

Spec = namedtuple("Spec", "n dim storage metric M ef data seed", defaults=("f32", "l2sq", 16, 64, None, None))
Shard = namedtuple("Shard", "ix ox gmap spec")


def _oracle_graph(oracle, ix, spec):
    p, zero, upper = ix.export_graph()
    return oracle.from_graph(oracle.Graph(p, zero, upper, spec.M, spec.ef)), (p, zero, upper)


def _rows(spec, i):
    return datagen.sift_shaped(spec.n, spec.dim, spec.data if spec.data is not None else 500 + 17 * i + spec.dim)


def _shard(abi, oracle, spec, i, offset):
    """Shard i of a call: built on the GPU (an empty or one-point shard: adopted with from_graph), its graph adopted by the oracle
    (bf16: the exported, rounded rows; cosine: the normalised rows), its PointIds mapped to global ids from `offset` on."""
    from instant_distance_b200 import sharded

    M, dim = spec.M, spec.dim
    if spec.n <= 1:
        pts = _rows(spec, i)
        if spec.metric == "cosine":
            pts = abi.normalize(pts) if spec.n else pts
        zero = np.full((spec.n, 2 * M), 0xFFFFFFFF, np.uint32)
        ix = abi.Index.from_graph(pts, zero, [], M, ef_search=spec.ef, storage=spec.storage, metric=spec.metric)
        local = np.arange(spec.n, dtype=np.uint32)
    else:
        kw = {"ml": 0.5} if M == 2 else {}
        seed = spec.seed if spec.seed is not None else 40 + i
        ix, local = abi.Index.build(_rows(spec, i), M=M, ef_search=spec.ef, seed=seed, storage=spec.storage, metric=spec.metric, **kw)
    ox = _oracle_graph(oracle, ix, spec)[0] if spec.n else None
    gmap = sharded.global_id_map(local, offset)
    ix.set_id_map(gmap)
    return Shard(ix, ox, gmap, spec)


def _shards(abi, oracle, specs):
    """Global ids run opposite to list order: the last shard holds the lowest."""
    offs = np.cumsum([0] + [s.n for s in specs[::-1]])[::-1][1:]
    return [_shard(abi, oracle, s, i, int(o)) for i, (s, o) in enumerate(zip(specs, offs))]


def _oracle_keys(oracle, sh, q, ef, k):
    """The shard's `nearest` list as K1's keys epilogue packs it: (distance bits << 32 | global id), empty slots all ones.
    Returns (keys nq x k, the oracle's per-layer counters)."""
    nq = len(q)
    if sh.ox is None:
        return np.full((nq, k), ms.KEY_NONE, dtype=np.uint64), None
    qq = cosine_ref.normalize(oracle, q) if sh.spec.metric == "cosine" else q
    ids, dist, lens, cnt = sh.ox.search(qq, ef_search=min(ef, sh.spec.n), k=k, counters=True, threads=THREADS)
    real = np.arange(k)[None, :] < np.minimum(lens, k)[:, None]
    gid = sh.gmap[np.where(real, ids, 0)].astype(np.uint64)
    keys = (np.ascontiguousarray(dist).view(np.uint32).astype(np.uint64) << np.uint64(32)) | gid
    keys[~real] = np.uint64(ms.KEY_NONE)
    return keys, cnt


def _same(got, want, what):
    ids, dist, lens = got
    assert (lens == want[2]).all(), f"{what}: lengths differ"
    bad = (ids != want[0]).any(axis=1)
    assert not bad.any(), f"{what}: ids differ in {bad.sum()} of {len(ids)} queries (first: {np.argmax(bad)})"
    assert dist.tobytes() == want[1].tobytes(), f"{what}: distance bytes differ"


def _check_fused(oracle, shards, got, q, ef_arg, k, what):
    """`got` = the fused result of `shards` for q: equal to the plain merge of the oracle's per-shard lists, and every shard ran the
    K1 cell of the dispatch statement with the oracle's per-layer counters.  Returns the per-shard keys."""
    keys = []
    for i, sh in enumerate(shards):
        ef = ef_arg or sh.spec.ef
        kk, cnt = _oracle_keys(oracle, sh, q, ef, k)
        keys.append(kk)
        cell = Cell(**sh.ix.last_kernel())
        if sh.ox is None:
            assert cell == Cell(0, 0, 0, 0, 0, 0, 0, 0), f"{what}: the empty shard {i} launched {cell}"
            continue
        want_cell = k1_cell(sh.spec.dim, sh.spec.M, ef, sh.spec.n, sh.spec.storage)
        assert cell == want_cell, f"{what}: shard {i} launched {cell}, the dispatch statement says {want_cell}"
        assert (sh.ix.last_counters(len(q)) == cnt).all(), f"{what}: shard {i}'s per-layer counters differ from the oracle's"
    _same(got, ms.merge(np.stack(keys), k, shards[0].spec.metric), what)
    return keys


def _fused(abi, oracle, comm, shards, q, ef_arg, k, what):
    got = abi.sharded_search_multi([s.ix for s in shards], comm, q, ef_search=ef_arg, k=k)
    return _check_fused(oracle, shards, got, q, ef_arg, k, what)


def _queries(shards, nq, kind, seed):
    q = datagen.sift_shaped(nq, shards[0].spec.dim, seed)
    if kind == "rows":  # half of them stored rows of the shards: distance 0, and exact ties where two shards hold the same row
        rows = [sh.ix.export_graph()[0] for sh in shards]
        for j in range(0, nq, 2):
            r = rows[(j // 2) % len(shards)]
            if len(r):
                q[j] = r[(7 * j) % len(r)]
    return q


Layout = namedtuple("Layout", "specs nq k ef queries", defaults=(64, 20, 64, "sift"))


def _three(dim, **kw):
    return [Spec(1200, dim, **kw)] * 3


LAYOUTS = {
    # the original three-shard cases: dim 48 (CH 1), the widest pre-merge of the old suite (3 x 100 keys per query)
    "dim48-k10-ef100": Layout([Spec(9000, 48, M=32, ef=100)] * 3, nq=1200, k=10, ef=100),
    "dim48-k100-ef100": Layout([Spec(9000, 48, M=32, ef=100)] * 3, nq=1200, k=100, ef=100),
    # one layout per K1 class, f32 and bf16 rows: CH 1, 2 (FULL at 256), 3, 6, 8 (FULL at 1024) and the long-row kernel
    **{f"{st}-dim{d}": Layout(_three(d, storage=st, M=16 if d % 2 else 32)) for d in (3, 100, 256, 300, 700, 1024, 1152)
       for st in ("f32", "bf16")},
    "cosine-dim100": Layout(_three(100, metric="cosine", M=24)),
    "cosine-bf16-dim1152": Layout(_three(1152, metric="cosine", storage="bf16")),
    "mixed-f32-bf16": Layout([Spec(1200, 100), Spec(1200, 100, "bf16"), Spec(1000, 100), Spec(900, 100, "bf16")]),
    # k and ef
    "k1": Layout(_three(64), k=1, ef=50),
    "k-eq-ef": Layout(_three(64), k=64, ef=64),
    "k-gt-ef": Layout(_three(64), k=50, ef=20),
    "k-gt-n": Layout([Spec(30, 64), Spec(1200, 64), Spec(45, 64)], k=64, ef=100),
    "ef10": Layout(_three(64), k=10, ef=10),
    "ef1024": Layout([Spec(2000, 64, M=32)] * 3, nq=48, k=100, ef=1024),
    "ef0-own-defaults": Layout([Spec(1200, 64, ef=40), Spec(1200, 64, ef=100), Spec(1200, 64, ef=250)], k=30, ef=0),
    # shards per call
    "one-shard": Layout([Spec(1500, 64)]),
    "two-shards": Layout([Spec(1500, 64), Spec(1300, 64)]),
    "eight-shards": Layout([Spec(400 + 50 * i, 32) for i in range(8)], k=16, ef=32),
    # shard edges
    "empty-shard": Layout([Spec(1200, 64), Spec(0, 64), Spec(1100, 64)], k=20),
    "one-point-shard": Layout([Spec(1200, 64), Spec(1, 64)], k=20),
    "same-rows-twice": Layout([Spec(1200, 64, data=9, seed=3), Spec(800, 64), Spec(1200, 64, data=9, seed=3)], k=15,
                              queries="rows"),
    "queries-are-rows": Layout(_three(64), k=20, queries="rows"),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_sharded_search_world_of_one(abi, oracle, comm, layout):
    """The fused path on one GPU against the plain merge of the oracle's per-shard lists; then shard 0 alone through the
    single-shard entry (K1 -> all-gather -> merge) against the plain merge of its own list."""
    L = LAYOUTS[layout]
    shards = _shards(abi, oracle, L.specs)
    q = _queries(shards, L.nq, L.queries, 77)
    keys = _fused(abi, oracle, comm, shards, q, L.ef, L.k, layout)
    if L.queries == "rows":
        assert (np.stack(keys) >> np.uint64(32) == 0).any(axis=(0, 2)).mean() >= 0.4, "queries equal to rows should find distance 0"
    if layout == "same-rows-twice":  # cross-shard exact ties, and the k boundary between the two keys of one tie
        d = np.stack(keys) >> np.uint64(32)
        assert (d[0] == d[2]).all()
        u = ms.merged_keys(np.stack(keys), L.k + 1) >> np.uint64(32)
        assert (u[:, L.k - 1] == u[:, L.k]).any()
    one = shards[0].ix.sharded_search(comm, q, ef_search=L.ef, k=L.k)
    _same(one, ms.merge(keys[0][None], L.k, shards[0].spec.metric), f"{layout}: shard 0 alone")
    [s.ix.close() for s in shards]


def test_large_batch(abi, oracle, comm):
    """20 000 queries: the pre-merge and the final merge run their grid-stride loops (their grids are capped at num_sms * 8
    blocks)."""
    _, num_sms = _device()
    nq = 20_000
    assert nq > num_sms * 8 * 4
    shards = _shards(abi, oracle, [Spec(600, 16, M=8, ef=24), Spec(500, 16, M=8, ef=24), Spec(700, 16, M=8, ef=24)])
    _fused(abi, oracle, comm, shards, _queries(shards, nq, "sift", 5), 24, 8, "20 000 queries")
    [s.ix.close() for s in shards]


def test_shard_counts_and_the_merge_limit(abi, oracle, comm):
    """1, 2, 8 and 64 shards in one call; 65 are refused.  k = 1024 over 28 shards fits the merge's shared memory (one warp per
    block), over 29 it is refused before anything is enqueued, and the same 29 shards then answer a call that fits."""
    max_smem, _ = _device()
    shards = [_shard(abi, oracle, Spec(60 + i, 8, M=4, ef=32), i, 200 * (64 - i)) for i in range(65)]
    q = datagen.sift_shaped(16, 8, 3)
    for n_local in (1, 2, 8, 64):
        _fused(abi, oracle, comm, shards[:n_local], q, 32, 10, f"{n_local} shards")
    with pytest.raises(abi.IdbError) as e:
        abi.sharded_search_multi([s.ix for s in shards], comm, q, ef_search=32, k=10)
    assert e.value.status == abi.ERR_INVALID_ARG
    assert ms.fits(28, 1024, max_smem) and ms.wpb(28, 1024, max_smem) == 1 and not ms.fits(29, 1024, max_smem)
    _fused(abi, oracle, comm, shards[:28], q, 32, 1024, "28 shards, k 1024")
    with pytest.raises(abi.IdbError) as e:
        abi.sharded_search_multi([s.ix for s in shards[:29]], comm, q, ef_search=32, k=1024)
    assert e.value.status == abi.ERR_UNSUPPORTED
    k = max_smem // (8 * 29)
    _fused(abi, oracle, comm, shards[:29], q, 32, k, f"29 shards, k {k} after the refusal")
    [s.ix.close() for s in shards]


def test_retry_pass_in_a_sharded_call(abi, oracle, comm, monkeypatch):
    """A 1024-slot hash set overflows in the main pass: every shard's retry pass re-runs its queries, keys included (through the id
    map), the result is still the plain merge, and the host entry does not report a capacity failure."""
    specs = [Spec(4000, 100, M=32, ef=100, seed=11 + i) for i in range(3)]
    built = _shards(abi, oracle, specs)
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    shards = []
    for sh in built:  # the same graphs, on indexes that read the environment above
        p, zero, upper = sh.ix.export_graph()
        ix = abi.Index.from_graph(p, zero, upper, sh.spec.M, ef_search=sh.spec.ef)
        ix.set_id_map(sh.gmap)
        shards.append(Shard(ix, sh.ox, sh.gmap, sh.spec))
        sh.ix.close()
    q = datagen.sift_shaped(64, 100, 21)
    _fused(abi, oracle, comm, shards, q, 100, 50, "retry")
    for i, sh in enumerate(shards):
        assert sh.ix.last_retried(0) > 0, f"shard {i} did not go through the retry pass"
    [s.ix.close() for s in shards]


@pytest.mark.parametrize("dim,metric", [(3, "l2sq"), (100, "l2sq"), (3, "cosine")])
def test_device_entry_equals_the_host_entry(abi, oracle, comm, dim, metric):
    """idb_sharded_search_batch_device_multi (torch buffers) gives the host entry's bytes, with the queries 16-byte aligned and one
    float off; dim 3 is not a multiple of 4.  Both pad the queries into the lane's buffer where K1 needs it."""
    import torch

    shards = _shards(abi, oracle, [Spec(900, dim, metric=metric), Spec(700, dim, metric=metric)])
    nq, k, ef = 200, 12, 40
    q = datagen.sift_shaped(nq, dim, 8)
    host = abi.sharded_search_multi([s.ix for s in shards], comm, q, ef_search=ef, k=k)
    _check_fused(oracle, shards, host, q, ef, k, f"host entry dim {dim}")
    for off in (0, 1):
        buf = torch.zeros(nq * dim + 4, dtype=torch.float32, device="cuda")
        buf[off:off + nq * dim] = torch.from_numpy(q.ravel()).cuda()
        ids = torch.empty((nq, k), dtype=torch.int32, device="cuda")
        dist = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        lens = torch.empty(nq, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        abi.sharded_search_multi_device([s.ix for s in shards], comm, buf.data_ptr() + 4 * off, nq, ef, k, ids.data_ptr(),
                                        dist.data_ptr(), lens.data_ptr())
        shards[0].ix.sync()
        got = (ids.cpu().numpy().view(np.uint32), dist.cpu().numpy(), lens.cpu().numpy().view(np.uint32))
        _same(got, host, f"device entry dim {dim} offset {off}")
    [s.ix.close() for s in shards]


def test_id_map_applies_to_a_plain_search(abi):
    """With a map set, a plain search returns map[pid] (bench.py compares global ids this way); None restores PointIds."""
    from instant_distance_b200 import sharded

    rows = datagen.sift_shaped(50, 16, 4)
    ix, local = abi.Index.build(rows, M=8, seed=2)
    q = datagen.sift_shaped(20, 16, 5)
    plain = ix.search(q, ef_search=64, k=60)  # k > n: padded slots stay INVALID
    gmap = sharded.global_id_map(local, 1_000_000)
    ix.set_id_map(gmap)
    mapped = ix.search(q, ef_search=64, k=60)
    want = np.where(plain[0] == 0xFFFFFFFF, 0xFFFFFFFF, gmap[np.minimum(plain[0], 49)])
    assert (plain[0] == 0xFFFFFFFF).any() and (mapped[0] == want).all()
    assert mapped[1].tobytes() == plain[1].tobytes() and (mapped[2] == plain[2]).all()
    ix.set_id_map(None)
    again = ix.search(q, ef_search=64, k=60)
    assert (again[0] == plain[0]).all() and again[1].tobytes() == plain[1].tobytes()
    ix.close()


def test_rejected_shard_lists(abi, comm):
    """A shard listed twice, and shards of different dims, are refused."""
    a, _ = abi.Index.build(datagen.sift_shaped(100, 16, 1), M=8)
    b, _ = abi.Index.build(datagen.sift_shaped(100, 16, 2), M=8)
    c, _ = abi.Index.build(datagen.sift_shaped(100, 20, 3), M=8)
    q = datagen.sift_shaped(4, 16, 4)
    for shards in ([a, b, a], [a, c]):
        with pytest.raises(abi.IdbError) as e:
            abi.sharded_search_multi(shards, comm, q, ef_search=16, k=4)
        assert e.value.status == abi.ERR_INVALID_ARG
    [x.close() for x in (a, b, c)]


@pytest.mark.skipif("_gpu_count() < 2", reason="needs >= 2 GPUs")
def test_sharded_search_two_ranks():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "scripts", "sharded_check.py"), "--points", "60000", "--queries", "3000"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("{")][-1]
    res = json.loads(line)
    assert res["local_eq_oracle"] and res["fused_eq_protocol"] and res["world"] == 2
