"""CPU statement of the exact range search (DESIGN.md §9b): the full exact ordering of every stored row for each query,
oracle.bruteforce(rows, q, k = n) (cosine: on the normalised queries, distances reported as 1 - cos, tests/cosine_ref.py), cut at
the radius.  The reported distance is monotone in the key's distance and NaN orders last, so the rows whose reported distance is
<= radius are a prefix of that ordering; `cut` takes that prefix and checks that nothing past it would have been kept.

Results are CSR like the library's: (offsets u64 [nq + 1], ids u32 [total], dist f32 [total])."""
import os

import numpy as np

from tests import cosine_ref


def full_order(oracle, rows, queries, metric="l2sq"):
    """(ids, reported distances), both nq x n: every stored row of each query in key order."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    q = np.ascontiguousarray(queries, dtype=np.float32)
    if q.ndim == 1:
        q = q[None, :]
    n = rows.shape[0]
    if n == 0:
        return np.zeros((q.shape[0], 0), np.uint32), np.zeros((q.shape[0], 0), np.float32)
    if metric == "cosine":
        ids, dist = oracle.bruteforce(rows, cosine_ref.normalize(oracle, q), n, threads=os.cpu_count() or 1)
        return ids, cosine_ref.reported(dist)
    return oracle.bruteforce(rows, q, n, threads=os.cpu_count() or 1)


def cut(ids, dist, radius, id_map=None):
    """The full orderings (ids, reported distances: nq x n) cut at `radius`, as CSR; ids through id_map after the cut."""
    with np.errstate(invalid="ignore"):
        keep = dist <= np.float32(radius)  # NaN is <= no radius
    counts = keep.sum(1)
    for i, c in enumerate(counts):  # the prefix property
        assert keep[i, :c].all(), f"query {i}: a kept row past the first {c}"
    offsets = np.zeros(ids.shape[0] + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(counts)
    out_ids = np.concatenate([ids[i, :c] for i, c in enumerate(counts)] + [np.zeros(0, np.uint32)]).astype(np.uint32)
    out_dist = np.concatenate([dist[i, :c] for i, c in enumerate(counts)] + [np.zeros(0, np.float32)]).astype(np.float32)
    if id_map is not None:
        out_ids = np.asarray(id_map, dtype=np.uint32)[out_ids]
    return offsets, out_ids, out_dist


def range_search(oracle, rows, queries, radius, metric="l2sq", id_map=None):
    """Every stored row (the rows as the index stores them: rounded, dequantised or normalised) within `radius` of each query."""
    ids, dist = full_order(oracle, rows, queries, metric)
    return cut(ids, dist, radius, id_map)
