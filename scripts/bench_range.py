"""Exact range search on one GPU: ms per call of idb_range_search_batch_device_lane at three radii, hits per query, the split between
its scan, offsets, gather + sort and finish kernels under torch.profiler, the exact k-NN search at k = 10 on the same queries, and
1 000 queries checked bit for bit against the CPU statement (tests/range_ref.py).

  python scripts/bench_range.py --out profiles/h100_range.json

Workloads: 1M x 128 sift-shaped f32 rows, squared L2, and 1M x 768 sift-shaped bf16 rows, cosine (tests/datagen.py), 10k queries
per call.  Radii: the median over the queries of the exact 10th, 100th and 1000th neighbour's distance (the exact search at
k = 1000 on the same queries), so a call returns about 10, 100 and 1000 hits per query.  The card's name, power limit and max SM
clock are read in the same call.
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

from tests import datagen, range_ref  # noqa: E402

RANKS = (10, 100, 1000)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def flat_index(abi, pts, storage, metric):
    zero = np.full((pts.shape[0], 4), 0xFFFFFFFF, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage, metric=metric)


def median(xs):
    return sorted(xs)[len(xs) // 2]


def kernel_split(prof):
    """Device microseconds per phase of one profiled range call."""
    us = {"scan": 0.0, "offsets": 0.0, "gather_sort": 0.0, "finish": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        key = ev.key
        if "range_scan_kernel" in key:
            us["scan"] += t
        elif "range_finish_kernel" in key:
            us["finish"] += t
        elif "range_gather_kernel" in key or any(w in key for w in ("SegmentedSort", "Partition", "Compact")):
            us["gather_sort"] += t
        elif "DeviceScan" in key or "scan" in key.lower():
            us["offsets"] += t
        elif "kernel" in key.lower() or "memset" in key.lower() or "memcpy" in key.lower():
            us["other"] += t
    return us


def time_range(torch, abi, ix, d_q, nq, radius, reps):
    """(offsets, ids, dist as numpy, result dict) of the device entry at this radius."""
    offsets = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    try:  # a counting call gives the total
        total = ix.range_search_device(d_q.data_ptr(), nq, radius, 0, offsets.data_ptr(), 0, 0)
    except abi.IdbError as e:
        if e.status != abi.ERR_CAPACITY:
            raise
        total = int(offsets[-1].item())
    ids = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(total, 1), dtype=torch.float32, device="cuda")

    def call():
        return ix.range_search_device(d_q.data_ptr(), nq, radius, total, offsets.data_ptr(), ids.data_ptr(), dist.data_ptr())

    call()  # warm-up: module load, occupancy query, scratch allocation, CUB's temporary storage
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()  # returns once the lane has run the call
        ms.append((time.perf_counter() - t0) * 1e3)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    h_off = offsets.cpu().numpy().view(np.uint64)
    counts = np.diff(h_off)
    r = {"radius": radius, "total_hits": total, "hits_per_query_mean": float(counts.mean()), "hits_per_query_max": int(counts.max()),
         "queries_without_hits": int((counts == 0).sum()), "ms_per_call": median(ms), "ms_all": ms,
         "profile_us": kernel_split(prof)}
    return h_off, ids.cpu().numpy().view(np.uint32)[:total], dist.cpu().numpy()[:total], r


def time_exact(torch, ix, d_q, nq, k, reps):
    ids = torch.empty(nq * k, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * k, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")

    def call():
        ix.exact_search_device(d_q.data_ptr(), nq, k, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=0)
        ix.sync()

    call()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        ms.append((time.perf_counter() - t0) * 1e3)
    return dist.cpu().numpy().reshape(nq, k), {"k": k, "ms_per_call": median(ms), "ms_all": ms}


def check_against_statement(O, stored, q, metric, runs_out, n):
    """The first queries of each radius's result against the CPU statement: oracle.bruteforce cut at the radius.  The statement
    needs only as many neighbours per query as the largest count plus one: its last column must lie past the radius."""
    nq = q.shape[0]
    k = min(n, max(int(np.diff(off[:nq + 1]).max()) for off, _, _, _ in runs_out) + 1)
    t0 = time.time()
    if metric == "cosine":
        from tests import cosine_ref

        ids, dist = O.bruteforce(stored, cosine_ref.normalize(O, q), k, threads=os.cpu_count() or 1)
        dist = cosine_ref.reported(dist)
    else:
        ids, dist = O.bruteforce(stored, q, k, threads=os.cpu_count() or 1)
    out = {"queries": nq, "k": k, "seconds": None, "passed": True, "per_radius": []}
    for off, g_ids, g_dist, radius in runs_out:
        full = k == n or bool((~(dist[:, -1] <= radius)).all())  # nothing past the k-th neighbour is a hit
        w_off, w_ids, w_dist = range_ref.cut(ids, dist, radius)
        m = int(off[nq])
        ok = full and off[:nq + 1].tobytes() == w_off.tobytes() and g_ids[:m].tobytes() == w_ids.tobytes() \
            and g_dist[:m].tobytes() == w_dist.tobytes()
        out["per_radius"].append({"radius": radius, "hits": m, "statement_covers_all_hits": full, "bytes_equal": bool(ok)})
        out["passed"] = out["passed"] and bool(ok)
    out["seconds"] = round(time.time() - t0, 1)
    return out


def workload(torch, abi, O, name, dim, storage, metric, a):
    pts = datagen.sift_shaped(a.n, dim, 1 if dim == 128 else 3)
    q = datagen.sift_shaped(a.nq, dim, 2 if dim == 128 else 4)
    ix = flat_index(abi, pts if metric == "l2sq" else abi.normalize(pts), storage, metric)
    del pts
    d_q = torch.from_numpy(q).cuda()
    res = {"workload": name, "shape": f"{a.n} x {dim} {storage} {metric}", "nq": a.nq}
    t0 = time.time()
    d1000, _ = time_exact(torch, ix, d_q, a.nq, max(RANKS), 1)
    res["radii_from_exact_k1000_s"] = round(time.time() - t0, 1)
    radii = [float(np.median(d1000[:, r - 1])) for r in RANKS]
    del d1000
    _, ex = time_exact(torch, ix, d_q, a.nq, 10, a.reps)
    res["exact_k10"] = ex
    res["runs"] = []
    kept = []
    for rank, radius in zip(RANKS, radii):
        off, ids, dist, r = time_range(torch, abi, ix, d_q, a.nq, radius, a.reps)
        r["neighbour_rank"] = rank
        r["ms_vs_exact_k10"] = r["ms_per_call"] / ex["ms_per_call"]
        res["runs"].append(r)
        kept.append((off, ids, dist, radius))
        print(json.dumps({"workload": name, **{k: v for k, v in r.items() if k != "ms_all"}}), flush=True)
    if a.check and storage == "f32":
        # the statement reads the rows as the index stores them
        stored = ix.export_graph()[0]
        res["statement_check"] = check_against_statement(O, stored, q[:a.check], metric, kept, a.n)
    del ix, d_q
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=1000, help="queries checked bit for bit against the CPU statement (f32 workload)")
    a = ap.parse_args()

    import torch

    from instant_distance_b200 import _abi as abi
    from oracle import oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = card()
    c["sms"] = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card": c, "n": a.n, "nq": a.nq, "workloads": []}
    res["workloads"].append(workload(torch, abi, O, "sift128-l2-f32", 128, "f32", "l2sq", a))
    res["workloads"].append(workload(torch, abi, O, "sift768-cosine-bf16", 768, "bf16", "cosine", a))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
