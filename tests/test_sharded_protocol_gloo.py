"""world_size-2 gloo test (CPU) of the sharded-search protocol (SURVEY §8e): contiguous input-range shards, per-shard
search, ONE all-gather of packed (distance, global id) keys, merge = exact k smallest of the union.
The per-shard searches are done by the CPU oracle here (the product has no CPU path); what is under test is the host
logic in instant_distance_b200.sharded, which the GPU path follows step for step."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import datagen, merge_statement


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n, dim, nq, k, ef, out):
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "instant-distance_b200", "python"))
    from instant_distance_b200 import sharded
    from oracle import oracle as O

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pts = datagen.uniform(n, dim, 5)
    q = datagen.uniform(nq, dim, 6)
    lo, hi = sharded.shard_range(n, rank, world)
    ix, local_ids = O.build(pts[lo:hi], seed=100 + rank)
    ids, d, lens = ix.search(q, ef_search=ef, k=k)
    gmap = sharded.global_id_map(local_ids, lo)
    gids = np.where(ids == 0xFFFFFFFF, 0, gmap[np.minimum(ids, hi - lo - 1)])
    keys = sharded.pack_keys(d, gids, np.minimum(lens, k))
    gathered = [torch.empty((nq, k), dtype=torch.int64) for _ in range(world)]
    dist.all_gather(gathered, torch.from_numpy(keys.view(np.int64)))  # the single collective
    all_keys = np.stack([g.numpy().view(np.uint64) for g in gathered])
    m_ids, m_dist, m_lens = sharded.merge_keys(all_keys, k)
    if rank == 0:
        np.savez(out, ids=m_ids, dist=m_dist, lens=m_lens)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_protocol_matches_single_process_union(tmp_path, oracle, world):
    from instant_distance_b200 import sharded

    n, dim, nq, k, ef = 3000, 16, 64, 10, 50
    out = str(tmp_path / "merged.npz")
    mp.spawn(_worker, args=(world, _free_port(), n, dim, nq, k, ef, out), nprocs=world, join=True)
    got = np.load(out)
    # single-process statement of the same thing: union of the per-shard results, exact k smallest by (dist, global id)
    pts = datagen.uniform(n, dim, 5)
    q = datagen.uniform(nq, dim, 6)
    cand = []
    for r in range(world):
        lo, hi = sharded.shard_range(n, r, world)
        ix, local_ids = oracle.build(pts[lo:hi], seed=100 + r)
        ids, d, lens = ix.search(q, ef_search=ef, k=k)
        inv = np.argsort(local_ids)  # pid -> local row
        cand.append((d, lo + inv[np.minimum(ids, hi - lo - 1)], lens))
    for qi in range(nq):
        pool = sorted((float(d[qi][j]), int(g[qi][j])) for d, g, lens in cand for j in range(min(int(lens[qi]), k)))[:k]
        assert [p[1] for p in pool] == got["ids"][qi].tolist()
        assert np.array([p[0] for p in pool], dtype=np.float32).tobytes() == got["dist"][qi].tobytes()
    # and the union recall is at least as good as brute force top-k restricted to what any shard saw
    bf, _ = oracle.bruteforce(pts, q, k)
    rec = np.mean([len(set(bf[i].tolist()) & set(got["ids"][i].tolist())) / k for i in range(nq)])
    assert rec > 0.9


def test_shard_ranges_partition_the_input():
    from instant_distance_b200 import sharded

    for n in (0, 1, 7, 1000, 10_000_000):
        for w in (1, 2, 3, 8):
            r = [sharded.shard_range(n, i, w) for i in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n and all(a[1] == b[0] for a, b in zip(r, r[1:]))


def test_merge_keys_pads_and_orders():
    from instant_distance_b200 import sharded

    d = np.array([[[0.5, 1.0, np.inf]], [[0.25, 1.0, 2.0]]], dtype=np.float32)
    g = np.array([[[7, 9, 0]], [[3, 2, 5]]], dtype=np.uint32)
    keys = np.stack([sharded.pack_keys(d[0], g[0], [2]), sharded.pack_keys(d[1], g[1], [3])])
    ids, dist, lens = sharded.merge_keys(keys, 4)
    assert ids.tolist() == [[3, 7, 2, 9]] and dist.tolist() == [[0.25, 0.5, 1.0, 1.0]] and lens.tolist() == [4]
    ids, dist, lens = sharded.merge_keys(keys, 6)
    assert ids[0].tolist() == [3, 7, 2, 9, 5, 0xFFFFFFFF] and lens.tolist() == [5] and np.isinf(dist[0][5])


@pytest.mark.parametrize("kind", merge_statement.KINDS + ("mixed",))
@pytest.mark.parametrize("G,nq,k", [(1, 5, 1), (2, 7, 2), (3, 9, 31), (7, 5, 33), (8, 4, 100), (64, 3, 32)])
def test_merge_keys_equals_the_plain_statement(kind, G, nq, k):
    """The host statement of the merge (sharded.merge_keys, used by the GPU tests and bench.py) against the plain one, on the
    adversarial key sets the merge kernel is checked on: ties across lists at the k boundary, empty and partial lists, unordered
    lists, distance bits 0 / subnormal / +inf / NaN and global ids 0 and 0xFFFFFFFE."""
    from instant_distance_b200 import sharded

    keys = merge_statement.mixed(G, nq, k, 7) if kind == "mixed" else merge_statement.keyset(kind, G, nq, k, 7)
    ids, dist, lens = sharded.merge_keys(keys, k)
    w_ids, w_dist, w_lens = merge_statement.merge(keys, k)
    assert (ids == w_ids).all() and dist.tobytes() == w_dist.tobytes() and (lens == w_lens).all()


def test_merge_key_sets_are_what_they_claim():
    """Keys are unique within a query, and each kind holds the cases it is there for."""
    ms = merge_statement
    for kind in ms.KINDS:
        keys = ms.keyset(kind, 3, 9, 5, 1)
        for q in range(9):
            real = [int(x) for x in keys[:, q, :].ravel() if int(x) != ms.KEY_NONE]
            assert len(set(real)) == len(real)
    prefix = ms.keyset("prefix", 3, 9, 5, 1)
    assert (prefix[:, 0, :] == np.uint64(ms.KEY_NONE)).all() and (prefix[:, 1, :] != np.uint64(ms.KEY_NONE)).all()
    ties = ms.keyset("ties", 3, 2, 5, 1)
    d, g = ties >> np.uint64(32), ties & np.uint64(0xFFFFFFFF)
    assert (d == d[:1, :, :1]).all() and (g[0].min(axis=1) > g[1].max(axis=1)).all()  # list 0 holds the highest ids
    special = ms.keyset("special", 2, 50, 8, 1)
    dbits = set((special >> np.uint64(32)).ravel().tolist())
    assert {0, ms.SUBNORMAL, ms.INF, ms.QNAN} <= dbits
    gids = special & np.uint64(0xFFFFFFFF)
    assert ((gids == 0).any(axis=(0, 2)) & (gids == 0xFFFFFFFE).any(axis=(0, 2))).all()
    # the cosine report halves the distance and keeps NaN and +inf
    keys = np.array([[(0x40000000 << 32) | 5, (ms.QNAN << 32) | 6, ms.KEY_NONE]], dtype=np.uint64)
    _, dist, lens = ms.report(keys, "cosine")
    assert dist.view(np.uint32).tolist() == [[0x3F800000, ms.QNAN, ms.INF]] and lens.tolist() == [2]
    _, dist, _ = ms.report(np.array([[(ms.SUBNORMAL << 32) | 1]], dtype=np.uint64), "cosine")
    assert dist.view(np.uint32).tolist() == [[0]]  # half the smallest subnormal rounds to even: 0


def test_merge_orders_exact_ties_by_global_id():
    """A shard orders exact-distance ties by its LOCAL PointId; the merged list is ordered by (distance, global id)."""
    from instant_distance_b200 import sharded

    d = np.array([[1.0, 2.0, 2.0]], dtype=np.float32)
    keys = np.stack([sharded.pack_keys(d, np.array([[5, 9, 4]], dtype=np.uint32), [3]),   # tie 9-before-4: local pid order
                     sharded.pack_keys(d + 10, np.array([[1, 2, 3]], dtype=np.uint32), [3])])
    ids, dist, lens = sharded.merge_keys(keys, 3)
    assert ids.tolist() == [[5, 4, 9]] and lens.tolist() == [3]
