"""CPU statement of the cosine metric (DESIGN.md §3a), built on the oracle's canonical squared L2 — the checker the GPU's cosine
results are compared with bit for bit.

Cosine is the canonical squared L2 between canonically normalised rows, and the reported distance is half of it.  So the oracle's
own squared-L2 build, search and brute force, run on the normalised rows and queries, are the cosine oracle; only the normalisation
and the halving are stated here:
  * normalize: s = the canonical sum of squares (oracle.l2sq against a zero row), r = sqrt(s), x / r — numpy's float32 sqrt and
    divide are correctly rounded, as __fsqrt_rn / __fdiv_rn are; s == 0 keeps the row zero; NaN results are written as 0x7fc00000;
  * reported: 0.5 * d in float32 (exact for normal floats), NaN kept as 0x7fc00000, +inf padding stays +inf.
"""
import numpy as np

QNAN = np.uint32(0x7FC00000)


def normalize(oracle, rows):
    x = np.ascontiguousarray(rows, dtype=np.float32)
    if x.ndim == 1:
        x = x[None, :]
    zeros = np.zeros(x.shape[1], np.float32)
    s = np.array([oracle.l2sq(r, zeros) for r in x], dtype=np.float32)
    r = np.sqrt(s)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(s[:, None] == 0, np.float32(0), x / r[:, None]).astype(np.float32)
    out.view(np.uint32)[np.isnan(out)] = QNAN
    return out


def reported(dist):
    d = np.ascontiguousarray(dist, dtype=np.float32)
    out = (np.float32(0.5) * d).astype(np.float32)
    out.view(np.uint32)[np.isnan(d)] = QNAN
    return out


def build(oracle, rows, **kw):
    """The cosine build: the oracle's build on the normalised rows.  Returns (Index, ids) like oracle.build."""
    return oracle.build(normalize(oracle, rows), **kw)


def search(oracle, index, queries, **kw):
    """index.search on the normalised queries, distances reported as cosine; counters (if asked for) unchanged."""
    res = list(index.search(normalize(oracle, queries), **kw))
    res[1] = reported(res[1])
    return tuple(res)


def bruteforce(oracle, points, queries, k, threads=1):
    ids, dist = oracle.bruteforce(normalize(oracle, points), normalize(oracle, queries), k, threads=threads)
    return ids, reported(dist)
