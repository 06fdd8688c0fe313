"""Insert throughput and the recall an insert gives up, on sift-shaped rows (M = 32, ef_construction = 100).

Times (host wall clock around each call, the device synchronised before and after, after a warm-up build and insert):
  * build of n - m points, then one insert of the other m points: points/s of each;
  * the same m points as `--calls` inserts;
  * one 1-row insert into the n-point index: one batch, its synchronisation and the screening-table rebuild over all rows;
  * the full build of n points;
recall@10 at ef_search = 100 against the exact search, for the full build, (n - m) + m and n/2 + n/2.
Two parts are taken apart:
  * the screening-table rebuild: the same 1-row insert into an n-point index built with IDB_SCREEN=0 (no table), the difference;
  * the per-batch synchronisation: under torch.profiler, the device idle time between the end of a batch's KA retry pass and the
    start of its K2 (`select_new_kernel`), for the insert (it reads KA's control block back in between) and for the build's layer-0
    batches (which read it after K2'), per batch.
Writes one JSON object to --out.
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

from instant_distance_b200 import _abi  # noqa: E402
from tests import datagen  # noqa: E402


def timed(fn):
    import torch

    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def recall(ix, q, truth):
    ids = ix.search(q, ef_search=100, k=10)[0]
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10.0 for a, b in zip(ids, truth)]))


def ka_k2_gaps(fn):
    """Runs fn under torch.profiler; per batch, microseconds from the end of the last insert_search_kernel before a
    select_new_kernel to that kernel's start."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                key=lambda e: e.time_range.start)
    gaps, last_ka_end = [], None
    for e in ev:
        if "insert_search_kernel" in e.name:
            last_ka_end = e.time_range.end
        elif "select_new_kernel" in e.name and last_ka_end is not None:
            gaps.append(e.time_range.start - last_ka_end)
            last_ka_end = None
    return gaps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--m", type=int, default=100_000)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = datagen.sift_shaped(a.n + a.nq, a.dim, 0)
    pts, q = rows[:a.n], rows[a.n:]
    n0 = a.n - a.m
    res = {"n": a.n, "m": a.m, "dim": a.dim, "M": 32, "ef_construction": 100}
    # warm-up: module load, device context, every kernel instantiation
    w, _ = _abi.Index.build(pts[:20_000], seed=1)
    w.insert(pts[20_000:30_000])
    del w
    ix, t_build = timed(lambda: _abi.Index.build(pts[:n0], seed=1)[0])
    _, t_ins = timed(lambda: ix.insert(pts[n0:]))
    res["build_s"], res["build_pts_per_s"] = t_build, n0 / t_build
    res["insert_one_call_s"], res["insert_one_call_pts_per_s"] = t_ins, a.m / t_ins
    ix2, _ = timed(lambda: _abi.Index.build(pts[:n0], seed=1)[0])
    step = a.m // a.calls
    ts = []
    for c in range(a.calls):
        _, t = timed(lambda: ix2.insert(pts[n0 + c * step:n0 + (c + 1) * step]))
        ts.append(t)
    res["insert_calls"] = a.calls
    res["insert_calls_s"] = ts
    res["insert_calls_pts_per_s"] = a.calls * step / sum(ts)
    _, t1 = timed(lambda: ix2.insert(pts[:1]))
    res["insert_1_row_s"] = t1  # one batch, its sync and the full screening-table rebuild over n + 1 rows
    del ix2
    os.environ["IDB_SCREEN"] = "0"
    ix3 = _abi.Index.build(pts[:a.n], seed=1)[0]
    del os.environ["IDB_SCREEN"]
    _, t1_noscreen = timed(lambda: ix3.insert(pts[:1]))
    del ix3
    res["insert_1_row_no_table_s"] = t1_noscreen
    res["table_rebuild_s"] = t1 - t1_noscreen
    # KA -> K2 gap per batch: 10 k rows into an n0-point index, and a build of 300 k points (its layer-0 batches)
    ix4 = _abi.Index.build(pts[:n0], seed=1)[0]
    g_ins = ka_k2_gaps(lambda: ix4.insert(pts[n0:n0 + step]))
    del ix4
    g_bld = ka_k2_gaps(lambda: _abi.Index.build(pts[:300_000], seed=1))
    res["ka_k2_gap_us_insert"] = {"batches": len(g_ins), "mean": float(np.mean(g_ins)) if g_ins else None,
                                  "max": float(np.max(g_ins)) if g_ins else None}
    big = g_bld[-8:]  # the build's last layer-0 batches: full-size batches, like the insert's
    res["ka_k2_gap_us_build_last8"] = {"batches": len(big), "mean": float(np.mean(big)) if big else None,
                                       "max": float(np.max(big)) if big else None}
    truth = ix.exact_search(q, k=10)[0]
    full, t_full = timed(lambda: _abi.Index.build(pts, seed=1)[0])
    res["full_build_s"], res["full_build_pts_per_s"] = t_full, a.n / t_full
    res["recall_full"] = recall(full, q, full.exact_search(q, k=10)[0])
    res["recall_build_n0_insert_m"] = recall(ix, q, truth)
    del full, ix
    half, _ = _abi.Index.build(pts[:a.n // 2], seed=1)
    half.insert(pts[a.n // 2:])
    res["recall_half_half"] = recall(half, q, half.exact_search(q, k=10)[0])
    try:
        import subprocess

        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
