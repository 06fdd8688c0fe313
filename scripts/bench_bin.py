"""bin row storage next to f32 and q8 (DESIGN.md §3d).  Sift-shaped rows, each element binarised at its column's median, indexed
once per storage with the same seed; the storages alternated --reps times in one call, on two workloads: 1M x 256 and 1M x 1024,
squared L2, ef_search = 100.  All three indexes hold the same 0/1 rows exactly (q8 stores a 0/1 row on the grid {0, 1}), so they
build the same graph and return the same results: the comparison is of the row formats alone, and each run checks that the ids and
distances equal the f32 index's.
Per storage and repetition:
  * build seconds (host clock around idb_build_ex, which returns after the device is done);
  * K1 ms per 10k-query batch (the library's CUDA events around K1; median of --batches) and queries/s of --batches batches issued
    back to back over lanes 0 and 1 (host clock around the loop, device synchronised; device-resident 0/1 queries and results);
  * candidate rows K1 fetched in full per query, and the fraction of queries the retry pass took again and that failed even there;
  * exact-search ms per call of --nq-exact queries (CUDA events);
  * resident bytes: rows, q8 row headers, screening table and graph.
Recall@10 is tie-aware (distances are integers, so ids at the 10th distance are interchangeable): a result counts when its distance
is at most the exact 10th distance of the bin index's own exact search, for 0/1 queries and for f32 queries (the sift queries mapped
into [0, 1] around the medians: the asymmetric distance).
The card's name, power limit and max SM clock are read in the same call.  Writes one JSON object to --out; --workload runs one of
them, and its result is added to an existing --out.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "instant-distance_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_q8 import card, time_exact, time_search  # noqa: E402
from instant_distance_b200 import _abi  # noqa: E402
from tests import datagen  # noqa: E402

WORKLOADS = [("bin256", 256), ("bin1024", 1024)]
STORAGES = ("f32", "bin", "q8")  # f32 first: the other two are compared with its results
EF = 100


def tie_recall(dist, exact10):
    """Tie-aware recall@10: the share of the 10 reported distances that are at most the exact 10th distance."""
    return float(np.mean(dist[:, :10] <= exact10[:, None]))


def overflows(torch, ix, d_q, nq):
    """(queries K1 left to the retry pass, queries that failed even there) of one device-resident search on lane 0."""
    ids = torch.empty(nq * 10, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * 10, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")
    ix.search_device(d_q.data_ptr(), nq, EF, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=0)
    ix.sync()
    return ix.last_retried(0), ix.last_failures(0)


def resident_bytes(ix, storage, dim, M=32):
    info = ix.info()
    n, nchunks = int(info.n), (dim + 3) // 4
    row = nchunks * {"f32": 16, "q8": 4, "bin": 1}[storage]
    table = 0 if storage in ("q8", "bin") else n * nchunks * 4 + 3 * nchunks * 16
    graph = n * 2 * M * 4 + sum(int(info.layer_n[l]) * M * 4 for l in range(1, int(info.n_layers)))
    out = {"rows": n * row, "headers": 8 * n if storage == "q8" else 0, "table": table, "graph": graph}
    out["total"] = sum(out.values())
    return out


def data(n, nq, dim):
    raw = datagen.sift_shaped(n + nq, dim, 11)
    med = np.median(raw[:n], axis=0)
    bits = (raw > med).astype(np.float32)
    sd = raw[:n].std(axis=0) + np.float32(1e-6)
    fq = np.clip((raw[n:] - med) / (4 * sd) + np.float32(0.5), 0, 1).astype(np.float32)
    return bits[:n], bits[n:], fq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nq-exact", type=int, default=10_000)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workload", choices=[w[0] for w in WORKLOADS], action="append")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    res = {"card": card(), "n": a.n, "nq": a.nq, "nq_exact": a.nq_exact, "batches": a.batches, "reps": a.reps, "M": 32,
           "ef_construction": 100, "ef_search": EF, "seed": 7, "workloads": {}}
    print(res["card"], flush=True)
    for name, dim in WORKLOADS:
        if a.workload and name not in a.workload:
            continue
        pts, q, fq = data(a.n, a.nq, dim)
        d_q = torch.from_numpy(q).cuda()
        d_fq = torch.from_numpy(fq).cuda()
        d_qe = torch.from_numpy(np.ascontiguousarray(q[:a.nq_exact])).cuda()
        w = {"dim": dim, "card": card(), "runs": []}
        base = None  # the f32 index's results, which every storage must equal
        for rep in range(a.reps):
            for storage in STORAGES:
                t = time.perf_counter()
                ix, _ = _abi.Index.build(pts, seed=7, storage=storage)
                build_s = time.perf_counter() - t
                retried, failed = overflows(torch, ix, d_q, a.nq)
                retried_f, failed_f = overflows(torch, ix, d_fq, a.nq)
                if failed or failed_f:  # the host-buffer search would raise IDB_ERR_CAPACITY
                    print(name, storage, "queries failed even the retry pass:", failed, failed_f, flush=True)
                    continue
                got = ix.search(q, ef_search=EF, k=10)
                full = ix.last_full_fetches() / len(q)
                got_f = ix.search(fq, ef_search=EF, k=10)
                k1_ms, qps = time_search(torch, ix, d_q, a.nq, EF, a.batches)
                exact_ms = time_exact(torch, ix, d_qe, a.nq_exact)
                r = {"rep": rep, "storage": storage, "build_s": build_s, "k1_ms_per_batch": k1_ms, "queries_per_s": qps,
                     "full_fetches_per_query": full, "retried_fraction": retried / len(q), "failed_fraction": failed / len(q),
                     "retried_fraction_f32_queries": retried_f / len(q), "failed_fraction_f32_queries": failed_f / len(q),
                     "exact_ms_per_call": exact_ms, "resident_bytes": resident_bytes(ix, storage, dim), "kernel": ix.last_kernel()}
                if storage == "bin" and "recall10_tie_aware" not in w:
                    ex = ix.exact_search(q, 10)[1][:, 9]
                    ex_f = ix.exact_search(fq, 10)[1][:, 9]
                    w["recall10_tie_aware"] = {"bin_queries": tie_recall(got[1], ex), "f32_queries": tie_recall(got_f[1], ex_f)}
                    w["distinct_rows"] = int(np.unique(np.packbits(pts != 0, axis=1), axis=0).shape[0])
                    print(name, "recall", w["recall10_tie_aware"], "distinct rows", w["distinct_rows"], flush=True)
                cur = (got[0], got[1].tobytes(), got_f[0], got_f[1].tobytes())
                if base is None and storage == "f32":
                    base = cur
                if base is not None:
                    r["identical_to_f32"] = bool((cur[0] == base[0]).all() and cur[1] == base[1] and (cur[2] == base[2]).all()
                                                 and cur[3] == base[3])
                print(name, json.dumps(r), flush=True)
                w["runs"].append(r)
                ix.close()
        for storage in STORAGES:
            rs = [r for r in w["runs"] if r["storage"] == storage]
            w[storage] = {k: [min(r[k] for r in rs), max(r[k] for r in rs)] for k in
                          ("build_s", "k1_ms_per_batch", "queries_per_s", "full_fetches_per_query", "retried_fraction",
                           "failed_fraction", "retried_fraction_f32_queries", "failed_fraction_f32_queries", "exact_ms_per_call")}
            w[storage]["resident_mb"] = {k: v / 1e6 for k, v in rs[0]["resident_bytes"].items()}
        res["workloads"][name] = w
        del d_q, d_fq, d_qe
        torch.cuda.empty_cache()
    if a.out and os.path.exists(a.out):
        with open(a.out) as f:
            prev = json.load(f)
        prev["workloads"].update(res["workloads"])
        res["workloads"] = prev["workloads"]
    text = json.dumps(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
