"""CPU statement of idb_index_remove (DESIGN.md §6b), in plain Python on the oracle.

remove(graph, pids, ef_construction=100, heuristic=True, keep_pruned=True) -> (Graph, new_ids)

graph: an oracle Graph (points as the index stores them, zero rows, upper rows).  For each layer L and each surviving point p of that
layer whose layer-L row lists a removed id, the candidates are the entries of p's row and of the layer-L rows of the removed ids it
lists (one hop), without p and without removed ids; W is the ef_construction smallest keys (canonical distance to points[p], PointId);
the new row is select_heuristic(p, W) (or the first 2M keys of W in simple mode), cut to M on an upper layer.  An entry is any value
but INVALID.  Then the PointIds are compacted in order: new(x) = x - |{r in R: r < x}|; the upper layers left empty are dropped.

The keys of a row's candidates come from one oracle.bruteforce call over the candidates in ascending PointId order: it orders by
(canonical distance, position), and positions follow PointIds, so its first min(ef, |C|) results are W.
"""
import numpy as np

from oracle import oracle as O

INVALID = 0xFFFFFFFF


def _row_ids(row):
    return row[row != INVALID]


def _repair_row(oracle_ix, points, p, row, layer_rows, removed, efc, heuristic, keep_pruned, M):
    cand = set(int(x) for x in _row_ids(row))
    for r in _row_ids(row):
        if removed[r]:
            cand.update(int(x) for x in _row_ids(layer_rows[r]))
    cand.discard(p)
    cand = np.array(sorted(x for x in cand if not removed[x]), dtype=np.uint32)
    if cand.size == 0:
        return np.zeros(0, np.uint32)
    k = min(efc, cand.size)
    pos, _ = O.bruteforce(points[cand], points[p], k)
    W = cand[pos[0]]
    if heuristic:
        out, _ = oracle_ix.select_heuristic(points[p], W, keep_pruned=keep_pruned)
    else:
        out = W[:2 * M]
    return np.asarray(out, dtype=np.uint32)


def repaired_rows(graph, pids, ef_construction=100, heuristic=True, keep_pruned=True):
    """The graph's layers after the repair and before the compaction: [zero, upper_1, ...] (copies), and the oracle index used."""
    points = np.ascontiguousarray(graph.points, dtype=np.float32)
    n, M = points.shape[0], graph.M
    removed = np.zeros(n, dtype=bool)
    removed[np.asarray(pids, dtype=np.int64)] = True
    ix = O.from_graph(graph)
    layers = [np.array(graph.zero, dtype=np.uint32, copy=True)] + [np.array(u, dtype=np.uint32, copy=True) for u in graph.upper]
    for rows in layers:
        before = rows.copy()  # repairs read their own row and removed rows only, which never change: the order of rows is free
        width = rows.shape[1]
        for p in range(rows.shape[0]):
            if removed[p]:
                continue
            ids = _row_ids(before[p])
            if not removed[ids].any():
                continue
            sel = _repair_row(ix, points, p, before[p], before, removed, ef_construction, heuristic, keep_pruned, M)[:width]
            rows[p, :] = INVALID
            rows[p, :sel.size] = sel
    return layers, removed


def remove(graph, pids, ef_construction=100, heuristic=True, keep_pruned=True):
    """Returns (Graph of the compacted index, new_ids: n entries, INVALID for a removed point)."""
    layers, removed = repaired_rows(graph, pids, ef_construction, heuristic, keep_pruned)
    n = removed.shape[0]
    keep = ~removed
    new_ids = np.full(n, INVALID, dtype=np.uint32)
    new_ids[keep] = np.arange(int(keep.sum()), dtype=np.uint32)

    def relabel(rows):
        kept = rows[keep[:rows.shape[0]]]
        return np.where(kept == INVALID, np.uint32(INVALID), new_ids[np.where(kept == INVALID, 0, kept)]).astype(np.uint32)

    zero = relabel(layers[0]).reshape(-1, 2 * graph.M)
    upper = [relabel(u).reshape(-1, graph.M) for u in layers[1:]]
    upper = [u for u in upper if u.shape[0] > 0]  # n_l' is non-increasing: the dropped layers are the top ones
    pts = np.ascontiguousarray(np.asarray(graph.points, dtype=np.float32)[keep])
    return O.Graph(pts, zero, upper, graph.M, graph.ef_search), new_ids
