"""Removal cost and what a removal leaves, on sift-shaped rows (1M x 128, M = 32, ef_construction = 100).

For each share removed (1 %, 10 %, 50 %, a random set each), on a fresh build of the same n points:
  * the time of one idb_index_remove call (host wall clock, the device synchronised before and after; after a warm-up removal on a
    smaller index, so the module and every kernel the call launches are loaded);
  * the rows repaired (surviving rows, over all layers, that listed a removed id) and the rows left empty (layer-0 rows with no entry
    afterwards), from the exported graphs;
  * recall@10 at ef_search = 100 of held-out queries against the exact search over the survivors, beside the same figure for a fresh
    build of the survivors;
  * the self-hit rate: the share of points whose own row, searched at k = 1 (ef_search = 100), returns the point itself, before and
    after.
Then, in a separate run under torch.profiler, the kernel time of one 10 % removal split into the repair (repair_kernel), the
compaction (keep flags, CUB's scan, the row copy and relabelling) and the screening-table rebuild (code_* kernels).
Writes one JSON object to --out.
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

INVALID = _abi.INVALID


def timed(fn):
    import torch

    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10.0 for a, b in zip(ids, truth)]))


def self_hits(ix, pts):
    ids = ix.search(pts, ef_search=100, k=1)[0][:, 0]
    return float(np.mean(ids == np.arange(len(pts), dtype=np.uint32)))


def repaired_rows(zero, upper, removed):
    count = 0
    for rows in [zero] + upper:
        hit = np.zeros(rows.shape[0], bool)
        valid = rows != INVALID
        hit[:] = (valid & removed[np.where(valid, rows, 0)]).any(axis=1)
        count += int((hit & ~removed[:rows.shape[0]]).sum())
    return count


def kernel_split(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"repair_ms": 0.0, "compaction_ms": 0.0, "table_rebuild_ms": 0.0, "other_ms": 0.0}
    names = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ms = (e.time_range.end - e.time_range.start) / 1000.0
        names[e.name[:80]] = names.get(e.name[:80], 0.0) + ms
        if "repair_kernel" in e.name:
            split["repair_ms"] += ms
        elif any(k in e.name for k in ("keep_flags", "drop_removed", "compact_rows", "relabel_rows", "DeviceScan", "Scan")):
            split["compaction_ms"] += ms
        elif "code_" in e.name:
            split["table_rebuild_ms"] += ms
        else:
            split["other_ms"] += ms
    split["by_name_ms"] = dict(sorted(names.items(), key=lambda kv: -kv[1]))
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--shares", default="0.01,0.1,0.5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"n": a.n, "dim": a.dim, "M": 32, "ef_construction": 100, "nq": a.nq}
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    rows = datagen.sift_shaped(a.n + a.nq, a.dim, 0)
    pts, q = rows[:a.n], rows[a.n:]
    w, _ = _abi.Index.build(pts[:50_000], seed=1)  # warm-up
    w.remove(np.arange(0, 50_000, 10, dtype=np.uint32))
    del w
    rng = np.random.default_rng(1)
    res["calls"] = []
    for share in [float(s) for s in a.shares.split(",")]:
        ix, _ = _abi.Index.build(pts, seed=1)
        stored, zero, upper = ix.export_graph()
        pids = rng.choice(a.n, int(a.n * share), replace=False).astype(np.uint32)
        removed = np.zeros(a.n, bool)
        removed[pids] = True
        r = {"share": share, "removed": int(pids.size), "layers_before": 1 + len(upper)}
        r["self_hit_before"] = self_hits(ix, stored)
        r["rows_repaired"] = repaired_rows(zero, upper, removed)
        del zero, upper
        _, r["remove_s"] = timed(lambda: ix.remove(pids))
        surv, zero1, upper1 = ix.export_graph()
        r["layers_after"] = 1 + len(upper1)
        r["rows_left_empty"] = int((zero1 == INVALID).all(axis=1).sum())
        del zero1, upper1
        truth = ix.exact_search(q, k=10)[0]
        r["recall_after_remove"] = recall(ix.search(q, ef_search=100, k=10)[0], truth)
        r["self_hit_after"] = self_hits(ix, surv)
        del ix
        fresh, fresh_ids = _abi.Index.build(surv, seed=1)
        row_of = np.empty_like(fresh_ids)
        row_of[fresh_ids] = np.arange(fresh_ids.size, dtype=np.uint32)
        r["recall_fresh_build"] = recall(row_of[fresh.search(q, ef_search=100, k=10)[0]], truth)
        del fresh
        print(json.dumps(r), flush=True)
        res["calls"].append(r)
    ix, _ = _abi.Index.build(pts, seed=1)
    pids = rng.choice(a.n, a.n // 10, replace=False).astype(np.uint32)
    res["profile_10pct"] = kernel_split(lambda: ix.remove(pids))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
