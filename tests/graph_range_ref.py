"""CPU statement of the graph range search (DESIGN.md §9c).  For query q, radius r and search width ef:

  * seeds: nearest(q), the oracle's search of the same graph at ef with k = ef (oracle.from_graph of the index's exported graph, rows
    as the index stores them: rounded, dequantised or normalised; a cosine index's queries normalised), cut to the members whose
    reported distance is <= r;
  * closure: the smallest set H holding the seeds such that, with every p in H, every layer-0 neighbour x of p (the entries of
    zero[p] up to its first INVALID) whose reported distance is <= r is in H too — a plain worklist;
  * output: H in key order (distance, then PointId) as CSR with range_ref's conventions, ids through the id map after ordering.

The distances are range_ref.full_order's (every stored row's reported distance per query), so each hit's distance bytes are the exact
range search's, and H(q) is a subsequence of range_ref.range_search's result."""
import os
from collections import deque

import numpy as np

from tests import cosine_ref, range_ref

INVALID = 0xFFFFFFFF


def neighbours(zero, p):
    """The entries of zero[p] up to its first INVALID."""
    row = zero[p]
    stop = np.flatnonzero(row == INVALID)
    return row[: stop[0] if stop.size else row.size]


def closure(zero, seeds, hit, order="fifo"):
    """The smallest set holding the seeds that are hits and closed under 'a hit's layer-0 neighbour that is a hit'.  order: how the
    worklist is taken ("fifo", "lifo", "reversed": FIFO over each row read backwards, or "levels": all of one level's rows at
    once in numpy, for large indexes); the set does not depend on it."""
    if order == "levels":
        h = np.zeros(len(hit), dtype=bool)
        level = np.unique(np.asarray(seeds, dtype=np.int64))
        level = level[hit[level]]
        h[level] = True
        while level.size:
            rows = zero[level]
            rows = rows[np.cumprod(rows != INVALID, axis=1).astype(bool)].astype(np.int64)  # each row up to its first INVALID
            level = np.unique(rows[hit[rows] & ~h[rows]])
            h[level] = True
        return set(np.flatnonzero(h).tolist())
    h = set()
    work = deque()
    for p in seeds:
        p = int(p)
        if hit[p] and p not in h:
            h.add(p)
            work.append(p)
    while work:
        p = work.popleft() if order != "lifo" else work.pop()
        row = neighbours(zero, p)
        for x in (row[::-1] if order == "reversed" else row):
            x = int(x)
            if x not in h and hit[x]:
                h.add(x)
                work.append(x)
    return h


def seeds(oracle, rows, zero, upper, M, queries, ef, metric="l2sq"):
    """nearest(q) of every query: (ids nq x ef, lens nq), the oracle's search of the graph at ef with k = ef."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    q = np.ascontiguousarray(queries, dtype=np.float32)
    if q.ndim == 1:
        q = q[None, :]
    if rows.shape[0] == 0 or ef == 0:
        return np.zeros((q.shape[0], max(ef, 1)), np.uint32), np.zeros(q.shape[0], np.uint32)
    ix = oracle.from_graph(oracle.Graph(rows, zero, upper, M, ef))
    if metric == "cosine":
        q = cosine_ref.normalize(oracle, q)
    ids, _, lens = ix.search(q, ef_search=ef, k=ef, threads=os.cpu_count() or 1)
    return ids, lens


def graph_range_search(oracle, rows, zero, upper, M, queries, radius, ef, metric="l2sq", id_map=None, order="fifo", full=None):
    """The graph range search over the index (rows as stored, its layer 0 `zero` and upper layers) at radius and ef, as CSR.
    full: range_ref.full_order's (ids, dist) when the caller has them already, or any prefix of each query's key order that holds
    every point within the radius (a point it does not list is no hit; rows shorter than the others end in INVALID ids)."""
    zero = np.ascontiguousarray(zero, dtype=np.uint32)
    ids, dist = full if full is not None else range_ref.full_order(oracle, rows, queries, metric)
    s_ids, s_lens = seeds(oracle, rows, zero, upper, M, queries, ef, metric)
    nq, n = ids.shape[0], np.asarray(rows).shape[0]
    keep = np.zeros(ids.shape, dtype=bool)
    for i in range(nq):
        listed = ids[i] != INVALID
        by_pid = np.full(n, np.nan, np.float32)
        by_pid[ids[i][listed]] = dist[i][listed]
        with np.errstate(invalid="ignore"):
            hit = by_pid <= np.float32(radius)  # NaN is <= no radius
        h = closure(zero, s_ids[i, : s_lens[i]], hit, order)
        keep[i] = listed & np.isin(ids[i], np.fromiter(h, dtype=np.int64, count=len(h)))
    counts = keep.sum(1)
    offsets = np.zeros(nq + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(counts)
    out_ids = np.concatenate([ids[i][keep[i]] for i in range(nq)] + [np.zeros(0, np.uint32)]).astype(np.uint32)
    out_dist = np.concatenate([dist[i][keep[i]] for i in range(nq)] + [np.zeros(0, np.float32)]).astype(np.float32)
    if id_map is not None:
        out_ids = np.asarray(id_map, dtype=np.uint32)[out_ids]
    return offsets, out_ids, out_dist
