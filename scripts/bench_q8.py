"""q8 row storage next to f32 and bf16 (DESIGN.md §3c): the same rows and seed built as one index per storage, the storages
alternated --reps times in one call, on two workloads:
  * 1M x 128 sift-shaped, squared L2, ef_search = 100;
  * 1M x 768 sift-shaped, cosine, ef_search = 128.
Per storage and repetition:
  * build seconds (host clock around idb_build_ex, which returns after the device is done);
  * K1 ms per 10k-query batch (the library's CUDA events around K1, idb_index_set_profiling; median of --batches) and queries/s
    of --batches batches issued back to back over lanes 0 and 1 (host clock around the loop, device synchronised; device-resident
    queries and results);
  * recall@10 at the workload's ef against the exact search of the f32 index (the user's ground truth; the same seed gives every
    storage the same PointIds) and against the index's own exact search;
  * exact-search ms per call of --nq-exact queries (CUDA events);
  * the candidate rows K1 fetched in full per query (a q8 index has no screening table, so it fetches every one);
  * resident bytes: rows, q8 row headers, screening table (codes and parameters) and graph (layer 0 and the upper layers).
On the cosine workload, the worst |sum x~^2 - 1| over the q8 index's stored (dequantised) rows.
The card's name, power limit and max SM clock are read in the same call, and stored with each workload.  Writes one JSON object to
--out; --workload runs one of them, and its result is added to an existing --out (one call per workload keeps each call short).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "instant-distance_b200", "python"))

from instant_distance_b200 import _abi  # noqa: E402
from tests import datagen  # noqa: E402

WORKLOADS = [("sift128-l2", 128, "l2sq", 100), ("sift768-cosine", 768, "cosine", 128)]
STORAGES = ("f32", "bf16", "q8")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def recall(got, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10.0 for a, b in zip(got, truth)]))


def time_search(torch, ix, d_q, nq, ef, batches):
    """(K1 ms per batch, queries/s): K1 from the library's events, one batch at a time; then queries/s of `batches` batches issued
    back to back, alternating lanes 0 and 1 (profiling off), host clock around the loop with the device synchronised."""
    bufs = [(torch.empty(nq * 10, dtype=torch.int32, device="cuda"), torch.empty(nq * 10, dtype=torch.float32, device="cuda"),
             torch.empty(nq, dtype=torch.int32, device="cuda")) for _ in range(2)]

    def call(lane):
        ids, dist, lens = bufs[lane]
        ix.search_device(d_q.data_ptr(), nq, ef, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=lane)

    for i in range(4):  # warm-up: both lanes' scratch, and the first launches of the process
        call(i % 2)
    ix.sync()
    ix.set_profiling(True)
    k1 = []
    for _ in range(batches):
        call(0)
        k1.append(ix.last_kernel_ms()[0])
    ix.set_profiling(False)
    ix.sync()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for i in range(batches):
        call(i % 2)
    ix.sync()
    return float(np.median(k1)), nq * batches / (time.perf_counter() - t)


def resident_bytes(ix, storage, dim, M=32):
    """What the index keeps on the device for its rows, their headers, the screening table and the graph."""
    info = ix.info()
    n, nchunks = int(info.n), (dim + 3) // 4
    row = nchunks * 4 * {"f32": 4, "bf16": 2, "f16": 2, "q8": 1}[storage]
    table = 0 if storage == "q8" else n * nchunks * 4 + 3 * nchunks * 16
    graph = n * 2 * M * 4 + sum(int(info.layer_n[l]) * M * 4 for l in range(1, int(info.n_layers)))
    out = {"rows": n * row, "headers": 8 * n if storage == "q8" else 0, "table": table, "graph": graph}
    out["total"] = sum(out.values())
    return out


def worst_unit_error(rows, chunk=65536):
    """max over the non-zero rows of |sum x^2 - 1|, in f64."""
    worst = 0.0
    for r0 in range(0, len(rows), chunk):
        s = np.einsum("ij,ij->i", rows[r0:r0 + chunk].astype(np.float64), rows[r0:r0 + chunk].astype(np.float64))
        s = s[s != 0]
        if len(s):
            worst = max(worst, float(np.abs(s - 1.0).max()))
    return worst


def time_exact(torch, ix, d_q, nq):
    ids = torch.empty(nq * 10, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * 10, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")
    stream = torch.cuda.ExternalStream(ix.lane_stream(0))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    ix.exact_search_device(d_q.data_ptr(), nq, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=0)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nq-exact", type=int, default=10_000)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", choices=[w[0] for w in WORKLOADS], action="append")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    res = {"card": card(), "n": a.n, "nq": a.nq, "nq_exact": a.nq_exact, "batches": a.batches, "reps": a.reps, "M": 32,
           "ef_construction": 100, "seed": 7, "workloads": {}}
    print(res["card"], flush=True)
    for name, dim, metric, ef in WORKLOADS:
        if a.workload and name not in a.workload:
            continue
        rows = datagen.sift_shaped(a.n + a.nq, dim, 11)
        pts, q = rows[:a.n], rows[a.n:]
        d_q = torch.from_numpy(q).cuda()
        d_qe = torch.from_numpy(np.ascontiguousarray(q[:a.nq_exact])).cuda()
        w = {"dim": dim, "metric": metric, "ef_search": ef, "card": card(), "runs": []}
        truth = None  # the f32 index's exact top 10
        for rep in range(a.reps):
            for storage in STORAGES:
                t = time.perf_counter()
                ix, _ = _abi.Index.build(pts, seed=7, metric=metric, storage=storage)
                build_s = time.perf_counter() - t
                own = ix.exact_search(q, 10)[0]
                if truth is None:
                    assert storage == "f32"
                    truth = own
                got = ix.search(q, ef_search=ef, k=10)[0]
                k1_ms, qps = time_search(torch, ix, d_q, a.nq, ef, a.batches)
                ix.search(q, ef_search=ef, k=10)
                full = ix.last_full_fetches() / len(q)
                exact_ms = time_exact(torch, ix, d_qe, a.nq_exact)
                r = {"rep": rep, "storage": storage, "build_s": build_s, "k1_ms_per_batch": k1_ms, "queries_per_s": qps,
                     "recall10_vs_f32_exact": recall(got, truth), "recall10_vs_own_exact": recall(got, own),
                     "exact_ms_per_call": exact_ms, "full_fetches_per_query": full, "resident_bytes": resident_bytes(ix, storage, dim),
                     "kernel": ix.last_kernel()}
                if storage == "q8" and metric == "cosine" and rep == 0:
                    w["q8_worst_unit_error"] = worst_unit_error(ix.export_graph()[0])
                    print(name, "q8 worst |sum x~^2 - 1|", w["q8_worst_unit_error"], flush=True)
                print(name, json.dumps(r), flush=True)
                w["runs"].append(r)
                ix.close()
        for storage in STORAGES:
            rs = [r for r in w["runs"] if r["storage"] == storage]
            w[storage] = {k: [min(r[k] for r in rs), max(r[k] for r in rs)] for k in
                          ("build_s", "k1_ms_per_batch", "queries_per_s", "recall10_vs_f32_exact", "recall10_vs_own_exact",
                           "exact_ms_per_call", "full_fetches_per_query")}
            w[storage]["resident_bytes"] = rs[0]["resident_bytes"]
        res["workloads"][name] = w
        del d_q, d_qe
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
