"""Batched GPU builds against the CPU statement of the batch schedule (oracle.build_batched, DESIGN.md §6), bit for bit.

Every caller of the library (idb_build_*, the instant_distance module, lib/idb_build_graph, bench.py) builds with batches of
concurrent inserts.  The schedule is deterministic, so a batched GPU graph must equal the statement's graph exactly: same
ids, stored rows, zero rows and upper layers.  The cases cover the KA / K2 / K2' instantiations (dim, M, ef_construction),
the schedule knobs, hub rows that need several re-prune rounds, bf16 storage and cosine, the execution knobs that must not
change results, and real batch sizes.  Each case asserts, from the statement's counters, that it reached the path it is for.
"""
import os
import time

import numpy as np
import pytest

from tests import cosine_ref, datagen

pytestmark = pytest.mark.gpu


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
    """(max_batch, growth) as build.cu takes them: insert_batch, else IDB_BUILD_MAXBATCH / IDB_BUILD_GROWTH, else 16384 / 8."""
    if insert_batch:
        return insert_batch, 8
    return (max(1, int(os.environ.get("IDB_BUILD_MAXBATCH", "16384"))), max(1, int(os.environ.get("IDB_BUILD_GROWTH", "8"))))


def _first_diff(name, got, want, st):
    bad = np.nonzero((got != want).any(axis=1))[0]
    if len(bad) == 0:
        return
    pid = int(bad[0])
    b = int(st["row_batch"][pid])
    g0, cnt = (int(x) for x in st["bounds"][b])
    pytest.fail(f"{name}: {len(bad)} rows differ; first PointId {pid}, last written in batch {b} (inserts [{g0}, {g0 + cnt}))\n"
                f"  gpu       {got[pid].tolist()}\n  statement {want[pid].tolist()}")


def _check(abi, oracle, rows, insert_batch=0, metric="l2sq", storage="f32", **kw):
    """Build on the GPU and with the statement; assert the graphs are identical.  Returns the statement's counters."""
    stmt = cosine_ref.normalize(oracle, rows) if metric == "cosine" else rows
    stmt = bf16_round(stmt) if storage == "bf16" else stmt
    max_batch, growth = _schedule(insert_batch)
    ix_o, ids_o, st = oracle.build_batched(stmt, max_batch, growth, threads=min(32, os.cpu_count() or 8), **kw)
    g = ix_o.export()
    ix_g, ids_g = abi.Index.build(rows, insert_batch=insert_batch, metric=metric, storage=storage, **kw)
    p, zero, upper = ix_g.export_graph()
    ix_g.close()
    assert (ids_g == ids_o).all(), "shuffle differs"
    assert p.tobytes() == g.points.tobytes(), "stored rows differ"
    _first_diff("zero layer", zero, g.zero, st)
    assert len(upper) == len(g.upper)
    for l, (a, b) in enumerate(zip(upper, g.upper), 1):
        assert a.shape == b.shape, (l, a.shape, b.shape)
        assert (a == b).all(), f"upper layer {l} differs (its zero rows agree): first PointId {np.nonzero((a != b).any(axis=1))[0][0]}"
    assert st["max_batch"] > 1 and st["link_requests"] > 0 and st["targets"] > 0, st
    return st


def _multi(st):
    """Every batched case has rounds with several new ids: the path insert_batch = 1 never takes."""
    assert st["multi_new_rounds"] > 0 or st["simple_multi_targets"] > 0, st


# ---- shapes across instantiations ----------------------------------------------------------------------------------

@pytest.mark.parametrize("gen,n,dim,kw", [
    (datagen.uniform, 3000, 2, {}),
    (datagen.uniform, 3000, 16, {}),
    (datagen.sift_shaped, 3000, 128, {}),
    (datagen.uniform, 2000, 300, {"M": 24}),
    (datagen.uniform, 1500, 512, {}),
    (datagen.sift_shaped, 1500, 768, {}),
    (datagen.uniform, 1200, 1000, {"M": 16}),
    (datagen.uniform, 1000, 1100, {}),
    (datagen.sift_shaped, 800, 1536, {"M": 16}),
])
def test_dims(abi, oracle, gen, n, dim, kw):
    _multi(_check(abi, oracle, gen(n, dim, 100 + dim), seed=dim, **kw))


@pytest.mark.parametrize("M", [2, 8, 16, 24, 32, 48, 64])
def test_M(abi, oracle, M):
    kw = {"ml": 0.5} if M == 2 else {}  # 1 / ln 2 > 1 is not a valid ml
    _multi(_check(abi, oracle, datagen.uniform(3000, 16, 200 + M), seed=M, M=M, **kw))


@pytest.mark.parametrize("efc", [1, 10, 100, 200, 400, 700])
def test_ef_construction(abi, oracle, efc):
    st = _check(abi, oracle, datagen.uniform(3000, 16, 300), seed=efc, M=16, ef_construction=efc)
    _multi(st)
    if efc <= 10:  # C = new ids + row prefix exceeds ef_construction: push admission rejects entries
        assert st["admission_limited_rounds"] > 0, st


def test_keep_pruned_off(abi, oracle):
    _multi(_check(abi, oracle, datagen.uniform(3000, 24, 400), seed=4, keep_pruned=0))


@pytest.mark.parametrize("dim", [2, 16])
def test_simple_mode(abi, oracle, dim):
    st = _check(abi, oracle, datagen.uniform(3000, dim, 500), seed=5, heuristic=0)
    assert st["simple_multi_targets"] > 0, st


# ---- schedules ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("insert_batch,n", [(0, 4000), (2, 4000), (7, 4000), (64, 4000), (1000, 12000)])
def test_insert_batch(abi, oracle, insert_batch, n):
    st = _check(abi, oracle, datagen.uniform(n, 16, 600), insert_batch=insert_batch, seed=6)
    _multi(st)
    if insert_batch:  # n is large enough for g0 / 8 to reach the cap
        assert st["max_batch"] == insert_batch


@pytest.mark.parametrize("env", [{"IDB_BUILD_GROWTH": "1"}, {"IDB_BUILD_MAXBATCH": "100"},
                                 {"IDB_BUILD_MAXBATCH": "300", "IDB_BUILD_GROWTH": "2"}])
def test_schedule_environment(abi, oracle, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    st = _check(abi, oracle, datagen.uniform(4000, 16, 700), seed=7)
    _multi(st)
    if "IDB_BUILD_MAXBATCH" in env:
        assert st["max_batch"] == int(env["IDB_BUILD_MAXBATCH"])


# ---- hubs and ties --------------------------------------------------------------------------------------------------

HUBS = {
    "duplicates": lambda: np.repeat(datagen.uniform(4, 8, 2), 2000, axis=0),  # 4 clusters of 2000 exact duplicates
    "grid_ties": lambda: datagen.grid_ties(8000, 3, 4, side=6),
    "sift_centers": lambda: datagen.sift_shaped(20000, 16, 4, centers=3),
}


@pytest.mark.parametrize("data", sorted(HUBS))
@pytest.mark.parametrize("heuristic", [1, 0])
def test_hubs_and_ties(abi, oracle, data, heuristic):
    st = _check(abi, oracle, HUBS[data](), seed=8, M=8, ef_construction=10, heuristic=heuristic)
    if heuristic:
        assert st["multi_new_rounds"] > 0 and st["admission_limited_rounds"] > 0, st
    else:
        assert st["simple_multi_targets"] > 0, st
    if data == "duplicates" or not heuristic:  # targets with more than kNewCap = 32 requests in one batch
        assert st["max_target_requests"] > 32, st
    if data == "duplicates" and heuristic:  # so their rows are re-pruned in several rounds
        assert st["multi_round_targets"] > 0, st


def test_hub_rows_in_several_rounds_at_default_parameters(abi, oracle):
    st = _check(abi, oracle, datagen.uniform(20000, 16, 4), seed=9)
    assert st["multi_round_targets"] > 0 and st["max_target_requests"] > 32, st


# ---- storage and metric ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gen,n,dim", [(datagen.sift_shaped, 5000, 128), (datagen.uniform, 1500, 768)])
def test_bf16_storage(abi, oracle, gen, n, dim):
    _multi(_check(abi, oracle, gen(n, dim, 800), storage="bf16", seed=10))


@pytest.mark.parametrize("storage", ["f32", "bf16"])
def test_cosine(abi, oracle, storage):
    _multi(_check(abi, oracle, datagen.sift_shaped(4000, 64, 900), metric="cosine", storage=storage, seed=11))


# ---- execution knobs that must not change results -------------------------------------------------------------------

def _stage_fits(M, dim, efc=100):
    """build.cu's IDB_BUILD_STAGE condition: SelectSmem::bytes(cand_cap, M, nchunks, stage=true) <= 56 KB."""
    cand_cap = max((efc + 31) // 32 * 32, 2 * M + 32)
    b = cand_cap * 8 + 2 * M * 4 + cand_cap * 4 + 2 * M * 4 + (2 * M + 32) * 4 + (2 * M + 32) * 8
    b = (b + 15) // 16 * 16 + 2 * M * ((dim + 3) // 4) * 16
    return b <= 56 * 1024


@pytest.mark.parametrize("M", [16, 32])
def test_staged_k2(abi, oracle, monkeypatch, M):
    """IDB_BUILD_STAGE=1: the kept rows of select_heuristic_warp are staged in shared memory (the kStage = true form)."""
    assert _stage_fits(M, 128)
    monkeypatch.setenv("IDB_BUILD_STAGE", "1")
    _multi(_check(abi, oracle, datagen.sift_shaped(5000, 128, 1000), seed=12, M=M))


@pytest.mark.parametrize("ctas", ["1", "16"])
def test_k2_grid(abi, oracle, monkeypatch, ctas):
    monkeypatch.setenv("IDB_BUILD_CTAS", ctas)
    _multi(_check(abi, oracle, datagen.sift_shaped(5000, 128, 1100), seed=13))


@pytest.mark.parametrize("tier", ["0", "1", "2"])
def test_visited_tier(abi, oracle, monkeypatch, tier):
    monkeypatch.setenv("IDB_VIS_TIER", tier)
    _multi(_check(abi, oracle, datagen.uniform(5000, 32, 1200), seed=14))


def test_retry_pass_hash_set(abi, oracle, monkeypatch):
    """A 1024-slot hash set cannot hold the ids these inserts visit: KA hands them to its retry pass (2^18 slots)."""
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    st = _check(abi, oracle, datagen.uniform(6000, 16, 1300), seed=15, ef_construction=200)
    assert st["max_insert_dist"] > 1024, st  # an insert evaluated more distinct ids on layer 0 than the table has slots


def test_retry_pass_and_b16_demotion(abi, oracle, monkeypatch):
    """b16 tables of 2048 bytes (64 buckets x 16 slots) overflow in KA: those inserts go through the retry pass, and once a batch
    has overflowed often enough, later batches use a larger visited flavour.  The graph must not change."""
    monkeypatch.setenv("IDB_B16_BYTES", "2048")
    st = _check(abi, oracle, datagen.uniform(6000, 16, 1400), seed=16, ef_construction=200)
    assert st["max_insert_dist"] > 64 * 16, st


# ---- scale ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gen,n,dim,kw", [
    (datagen.sift_shaped, 200_000, 128, {}),
    (datagen.uniform, 100_000, 300, {"M": 24, "ef_construction": 200}),  # BASELINE configs[2]'s build parameters
])
def test_scale(abi, oracle, gen, n, dim, kw):
    t = time.time()
    st = _check(abi, oracle, gen(n, dim, 1500), seed=17, **kw)
    print(f"{n} x {dim} {kw}: batches {st['batches']}, largest batch {st['max_batch']}, largest hub {st['max_target_requests']} "
          f"requests, {st['multi_round_targets']} multi-round targets, {time.time() - t:.1f} s")
    assert st["max_batch"] >= 10_000 and st["multi_round_targets"] > 0, st
