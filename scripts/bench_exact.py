"""Exact k-NN on one GPU: throughput of idb_exact_search_batch_device_lane, the split between its scan and merge kernels, its distance
to the FP32 issue bound and the byte bound, a bit-for-bit check against oracle.bruteforce, and the recall@10 of the default HNSW search
measured against this exact search and against bench.brute_force_topk_torch.

  python scripts/bench_exact.py --out profiles/h100_exact.json

Shapes: 1M x 128 sift-shaped f32 rows (tests/datagen.py) with 10k queries at k = 10 and k = 100, and 1M x 768 bf16 rows (the row
shape of BASELINE configs[3]) at k = 10.  Bounds are computed from shapes:
  FP32 issue bound = pairs x (2 dim + 3 dim / 4 + 31) FP32 instructions / (SMs x 128 lanes x max SM clock)
  byte bound       = ceil(nq / queries per CTA) x n x row bytes / 3.35 TB/s (every CTA streams its slice of rows from HBM once)
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "instant-distance_b200", "python"))

from tests import datagen  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
# queries per CTA of the scan kernel per CH cell (exact.cu: 8 warps x QW queries; the long-row kernel has QW = 1)
Q_PER_CTA = {1: 64, 2: 32, 3: 16, 4: 16, 6: 16, 8: 8, 0: 8}


def kernel_ch(dim):
    c = ((dim + 3) // 4 + 31) // 32
    return c if c <= 4 else 6 if c <= 6 else 8 if c <= 8 else 0


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def flat_index(abi, pts, storage):
    zero = np.full((pts.shape[0], 4), 0xFFFFFFFF, dtype=np.uint32)
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage)


def time_exact(torch, ix, d_q, nq, k, reps):
    ids = torch.empty(nq * k, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * k, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")
    stream = torch.cuda.ExternalStream(ix.lane_stream(0))

    def call():
        ix.exact_search_device(d_q.data_ptr(), nq, k, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=0)

    call()  # warm-up: module load, occupancy query, scratch allocation
    ix.sync()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    # kernel split in a separate, profiled call
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        ix.sync()
    scan_us = merge_us = other_us = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if "exact_scan_kernel" in ev.key:
            scan_us += t
        elif "merge_topk_kernel" in ev.key:
            merge_us += t
        elif "kernel" in ev.key.lower() or "memset" in ev.key.lower() or "memcpy" in ev.key.lower():
            other_us += t
    total = scan_us + merge_us + other_us
    return ids, dist, lens, {
        "ms_per_batch": sorted(ms)[len(ms) // 2], "ms_all": ms, "queries_per_s": nq / (sorted(ms)[len(ms) // 2] / 1e3),
        "profile_us": {"scan": scan_us, "merge": merge_us, "other": other_us},
        "merge_fraction": merge_us / total if total else None,
    }


def bounds(c, n, nq, dim, row_bytes):
    pairs = n * nq
    fp32_s = pairs * (2 * dim + 3 * dim / 4 + 31) / (c["sms"] * 128 * c["max_sm_clock_mhz"] * 1e6)
    byte_s = math.ceil(nq / Q_PER_CTA[kernel_ch(dim)]) * n * row_bytes / HBM_BYTES_PER_S
    return {"fp32_issue_bound_ms": fp32_s * 1e3, "byte_bound_ms": byte_s * 1e3, "binding": "fp32" if fp32_s >= byte_s else "bytes"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=1000, help="queries checked bit for bit against oracle.bruteforce")
    a = ap.parse_args()

    import torch

    import bench
    from instant_distance_b200 import _abi as abi
    from oracle import oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = card()
    c["sms"] = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card": c, "n": a.n, "nq": a.nq, "runs": []}

    # 1M x 128 f32, k = 10 and 100
    dim = 128
    pts = datagen.sift_shaped(a.n, dim, 1)
    q = datagen.sift_shaped(a.nq, dim, 2)
    ix = flat_index(abi, pts, "f32")
    d_q = torch.from_numpy(q).cuda()
    for k in (10, 100):
        ids, dist, _, r = time_exact(torch, ix, d_q, a.nq, k, a.reps)
        r.update(shape=f"{a.n} x {dim} f32", k=k, **bounds(c, a.n, a.nq, dim, dim * 4))
        r["fraction_of_fp32_bound"] = r["fp32_issue_bound_ms"] / r["ms_per_batch"]
        res["runs"].append(r)
        if k == 10:
            exact10 = ids.cpu().numpy().view(np.uint32).reshape(a.nq, k)
            d10 = dist.cpu().numpy().reshape(a.nq, k)
    t0 = time.time()
    o_ids, o_dist = O.bruteforce(pts, q[:a.check], 10, threads=os.cpu_count() or 1)
    res["oracle_check"] = {"queries": a.check, "k": 10, "seconds": round(time.time() - t0, 1),
                           "ids_equal": bool((exact10[:a.check] == o_ids).all()),
                           "distance_bytes_equal": d10[:a.check].tobytes() == o_dist.tobytes()}
    res["oracle_check"]["passed"] = res["oracle_check"]["ids_equal"] and res["oracle_check"]["distance_bytes_equal"]

    # recall@10 of the default HNSW search, against this exact search and against the torch brute force bench.py uses
    t0 = time.time()
    hnsw, perm = abi.Index.build(pts, seed=1)
    t_build = time.time() - t0
    by_pid = np.empty_like(perm)
    by_pid[perm] = np.arange(len(perm), dtype=perm.dtype)  # PointId -> input row
    approx, _, _ = hnsw.search(q, ef_search=0, k=10)
    approx_rows = by_pid[approx]
    t_ids, _ = bench.brute_force_topk_torch(torch.from_numpy(pts).cuda(), q, 10)
    res["recall_at_10_default_search"] = {
        "ef_search": int(hnsw.info().ef_search), "graph_build_s": round(t_build, 1),
        "vs_exact_search": bench.recall_at_k(approx_rows, exact10), "vs_torch_brute_force": bench.recall_at_k(approx_rows, t_ids),
        "torch_vs_exact_id_mismatches": int((np.sort(t_ids, 1) != np.sort(exact10, 1)).any(1).sum()),
    }
    del hnsw, ix, d_q
    torch.cuda.empty_cache()

    # 1M x 768 bf16, k = 10
    dim = 768
    pts = datagen.sift_shaped(a.n, dim, 3)
    q = datagen.sift_shaped(a.nq, dim, 4)
    ix = flat_index(abi, pts, "bf16")
    del pts
    d_q = torch.from_numpy(q).cuda()
    _, _, _, r = time_exact(torch, ix, d_q, a.nq, 10, max(1, a.reps - 1))
    r.update(shape=f"{a.n} x {dim} bf16", k=10, **bounds(c, a.n, a.nq, dim, dim * 2))
    r["fraction_of_fp32_bound"] = r["fp32_issue_bound_ms"] / r["ms_per_batch"]
    res["runs"].append(r)

    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
