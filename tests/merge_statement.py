"""Plain statement of the sharded search's merge (K4, `merge_topk_kernel` in csrc/sharded.cu), and the key sets it is checked on.

A key is (distance bits << 32 | global id); all ones is an empty slot.  For each query the merge takes the real keys of its G lists,
keeps the k smallest, and reports: the keys themselves (a rank's pre-merge), or ids = the low 32 bits, distances = the high 32 bits
reported in the index's metric (squared L2: as they are; cosine: 0.5 * d, with the NaN 0x7fc00000 kept as it is), padded with
0xFFFFFFFF / +inf, and len = how many real keys were kept.  The sort here is Python's on Python ints: nothing about floats or dtypes
enters the order.  `instant_distance_b200.sharded.merge_keys` is the host statement the GPU tests and bench.py use; the CPU tests
check it against this one.
"""
import numpy as np

KEY_NONE = 0xFFFFFFFFFFFFFFFF
QNAN = 0x7FC00000
INF = 0x7F800000
SUBNORMAL = 0x00000001
# distance bits that are legal in a key: 0, subnormals, normals, +inf and the canonical NaN (the largest)
SPECIAL_DIST = np.array([0, SUBNORMAL, 0x00000003, 0x007FFFFF, 0x00800000, 0x3F800000, INF, QNAN], dtype=np.uint64)


def merged_keys(all_keys, k):
    """all_keys: G x nq x kk u64 -> the merged keys, nq x k u64 (what a rank's pre-merge writes)."""
    all_keys = np.asarray(all_keys, dtype=np.uint64)
    G, nq, _ = all_keys.shape
    keys = np.full((nq, k), KEY_NONE, dtype=np.uint64)
    for q in range(nq):
        col = all_keys[:, q, :].ravel()
        kept = sorted(col[col != np.uint64(KEY_NONE)].tolist())[:k]
        keys[q, :len(kept)] = kept
    return keys


def report(keys, metric="l2sq"):
    """Merged keys (nq x k) -> (ids nq x k u32, dist nq x k f32, lens nq u32) as the final merge reports them."""
    real = keys != np.uint64(KEY_NONE)
    ids = np.where(real, keys & np.uint64(0xFFFFFFFF), 0xFFFFFFFF).astype(np.uint32)
    dbits = np.where(real, keys >> np.uint64(32), INF).astype(np.uint32)
    dist = dbits.view(np.float32).copy()
    if metric == "cosine":
        half = (np.float32(0.5) * dist).astype(np.float32)
        dist = np.where(dbits == QNAN, dist, half)
    elif metric != "l2sq":
        raise ValueError(metric)
    return ids, dist, real.sum(axis=1).astype(np.uint32)


def merge(all_keys, k, metric="l2sq"):
    """The final merge: (ids, dist, lens)."""
    return report(merged_keys(all_keys, k), metric)


def wpb(G, k, max_smem):
    """Warps per block of the merge launch (launch_merge): 4, halved while their G x k keys each do not fit max_smem."""
    w = 4
    while w > 1 and G * k * 8 * w > max_smem:
        w //= 2
    return w


def fits(G, k, max_smem):
    return G * k * 8 <= max_smem


# ---- key sets: keys unique within a query, as global ids are --------------------------------------------------------------

KINDS = ("random", "prefix", "ties", "special")


def _ids(rng, G, nq, k):
    """G x nq x k distinct ids per query: a fixed set of G*k distinct values below 2^30 XOR a per-query mask with bit 30 set (so
    never 0 or 0xFFFFFFFE, which `special` places itself)."""
    base = rng.choice(1 << 30, size=G * k, replace=False).astype(np.uint64).reshape(G, 1, k)
    mask = rng.integers(1 << 30, 1 << 31, size=nq, dtype=np.uint64)
    return base ^ mask[None, :, None]


def _dist(rng, shape):
    """Random finite distance bits; a quarter drawn from a few values, so that distances tie across lists."""
    d = rng.integers(0, INF, size=shape, dtype=np.uint64)
    pool = np.array([0x3F000000, 0x3F800000, 0x40000000, 0x40400000], dtype=np.uint64)
    pick = rng.random(shape) < 0.25
    d[pick] = pool[rng.integers(0, len(pool), size=int(pick.sum()))]
    return d


def _shuffle_lists(rng, keys):
    """Lists in no particular order: a shard orders exact ties by its local PointId, and the merge assumes no order at all."""
    return np.take_along_axis(keys, rng.random(keys.shape).argsort(axis=2), axis=2)


def keyset(kind, G, nq, k, seed):
    """G x nq x k u64 keys of one kind:
      random  random distances (a quarter of them tied across lists) and ids, lists unordered;
      prefix  lists that are prefixes of length 0..k (uniform, and every third query has no real key at all), then empty slots;
      ties    every key of a query at one distance, global ids running opposite to list order, so the k-th key of the merge (G > 1)
              falls inside the tie group;
      special distance bits 0, subnormal, normal, +inf and NaN, and global ids 0 and 0xFFFFFFFE in every query."""
    rng = np.random.default_rng(seed)
    shape = (G, nq, k)
    if kind == "ties":
        # list g holds ids descending in g: G-1-g blocks above list G-1's; inside a list, descending too
        rank = (G - 1 - np.arange(G))[:, None, None] * k + (k - 1 - np.arange(k))[None, None, :]
        ids = np.broadcast_to(rank, shape).astype(np.uint64) + rng.integers(0, 1 << 20, size=nq, dtype=np.uint64)[None, :, None]
        dist = np.broadcast_to(rng.choice(SPECIAL_DIST[:6], size=nq)[None, :, None], shape)
        return (dist << np.uint64(32)) | ids
    keys = (_dist(rng, shape) << np.uint64(32)) | _ids(rng, G, nq, k)
    if kind == "random":
        return keys
    if kind == "prefix":
        keys = np.sort(keys, axis=2)  # (a shard's list is ascending; empty slots only at its end)
        lens = rng.integers(0, k + 1, size=(G, nq))
        lens[:, ::3] = 0
        if nq > 1:
            lens[:, 1] = k  # one query with every list full
        keys[np.arange(k)[None, None, :] >= lens[:, :, None]] = np.uint64(KEY_NONE)
        return keys
    if kind == "special":
        d = SPECIAL_DIST[rng.integers(0, len(SPECIAL_DIST), size=shape)]
        keys = (d << np.uint64(32)) | (keys & np.uint64(0xFFFFFFFF))
        keys[0, :, 0] = (keys[0, :, 0] & np.uint64(0xFFFFFFFF00000000)) | np.uint64(0)
        keys[G - 1, :, k - 1] = (keys[G - 1, :, k - 1] & np.uint64(0xFFFFFFFF00000000)) | np.uint64(0xFFFFFFFE)
        return _shuffle_lists(rng, keys)
    raise ValueError(kind)


def mixed(G, nq, k, seed):
    """Every kind, query q taking kind q % 4 (each kind's own layout, on its share of the queries)."""
    out = np.empty((G, nq, k), dtype=np.uint64)
    for i, kind in enumerate(KINDS):
        qs = np.arange(i, nq, len(KINDS))
        if len(qs):
            out[:, qs, :] = keyset(kind, G, len(qs), k, seed + i)
    return out
