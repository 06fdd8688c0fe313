"""Graph range search on one GPU: ms per call of idb_graph_range_search_batch_device_lane at three radii and two search widths, hits
per query, recall against the exact range search (idb_range_search_batch_device_lane, timed in the same run), and 1 000 queries
checked bit for bit against the CPU statement (tests/graph_range_ref.py).

  python scripts/bench_graph_range.py --out profiles/h100_graph_range.json

Workload: 1M x 128 sift-shaped f32 rows (tests/datagen.py), squared L2, a graph built on the GPU (M = 32, ef_construction = 100), 10k
queries per call.  Radii: the median over the queries of the exact 10th, 100th and 1000th neighbour's distance (the exact search at
k = 1000 on the same queries), as scripts/bench_range.py chooses them.  ef_search = 100 and 200.  Each time is the median of three
calls after a warm-up, host clock around the device entry (which returns once its lane has run the call).  The card's name, power
limit and max SM clock are read in the same call.
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

from tests import datagen, graph_range_ref  # noqa: E402

RANKS = (10, 100, 1000)
EFS = (100, 200)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def median(xs):
    return sorted(xs)[len(xs) // 2]


def timed(torch, abi, device_call, nq, reps):
    """(offsets, ids, dist as numpy, ms list) of a range device entry device_call(capacity, offsets, ids, dist) -> total."""
    offsets = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
    try:  # a counting call gives the total
        total = device_call(0, offsets.data_ptr(), 0, 0)
    except abi.IdbError as e:
        if e.status != abi.ERR_CAPACITY:
            raise
        total = int(offsets[-1].item())
    ids = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
    dist = torch.empty(max(total, 1), dtype=torch.float32, device="cuda")

    def call():
        return device_call(total, offsets.data_ptr(), ids.data_ptr(), dist.data_ptr())

    call()  # warm-up: module load, scratch allocation, CUB's temporary storage
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        ms.append((time.perf_counter() - t0) * 1e3)
    return offsets.cpu().numpy().view(np.uint64), ids.cpu().numpy().view(np.uint32)[:total], dist.cpu().numpy()[:total], ms


def exact_k(torch, ix, d_q, nq, k):
    ids = torch.empty(nq * k, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * k, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")
    ix.exact_search_device(d_q.data_ptr(), nq, k, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=0)
    ix.sync()
    return dist.cpu().numpy().reshape(nq, k)


def recall(g_off, g_ids, e_off, e_ids):
    """Pooled (all graph hits / all exact hits) and the mean over queries with an exact hit; the graph hits are a subset."""
    gc, ec = np.diff(g_off).astype(np.int64), np.diff(e_off).astype(np.int64)
    per = gc[ec > 0] / ec[ec > 0]
    return {"pooled": float(gc.sum() / max(ec.sum(), 1)), "per_query_mean": float(per.mean()) if per.size else 1.0}


def is_subset(g_off, g_ids, e_off, e_ids, nq):
    for i in range(nq):
        g = g_ids[int(g_off[i]):int(g_off[i + 1])]
        e = e_ids[int(e_off[i]):int(e_off[i + 1])]
        if not np.isin(g, e).all():
            return False
    return True


def check_against_statement(O, stored, zero, upper, M, q, runs, exact_offsets):
    """The first queries of each run against the CPU statement.  The statement needs each query's key order only as far as the
    largest radius reaches: oracle.bruteforce with k = the most exact hits plus one, whose last column must lie past every radius."""
    nq = q.shape[0]
    t0 = time.time()
    k = min(stored.shape[0], max(int(np.diff(off[:nq + 1]).max()) for off in exact_offsets) + 1)
    ids, dist = O.bruteforce(stored, q, k, threads=os.cpu_count() or 1)
    out = {"queries": nq, "k": k, "passed": True, "per_run": []}
    for (ef, radius), (off, g_ids, g_dist) in runs.items():
        covers = k == stored.shape[0] or bool((~(dist[:, -1] <= radius)).all())
        w_off, w_ids, w_dist = graph_range_ref.graph_range_search(O, stored, zero, upper, M, q, radius, ef, order="levels", full=(ids, dist))
        m = int(off[nq])
        ok = covers and off[:nq + 1].tobytes() == w_off.tobytes() and g_ids[:m].tobytes() == w_ids.tobytes() \
            and g_dist[:m].tobytes() == w_dist.tobytes()
        out["per_run"].append({"ef_search": ef, "radius": radius, "hits": m, "statement_covers_all_hits": covers, "bytes_equal": bool(ok)})
        out["passed"] = out["passed"] and bool(ok)
    out["seconds"] = round(time.time() - t0, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=1000, help="queries checked bit for bit against the CPU statement")
    a = ap.parse_args()

    import torch

    from instant_distance_b200 import _abi as abi
    from oracle import oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = card()
    c["sms"] = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card": c, "n": a.n, "nq": a.nq, "workload": f"{a.n} x 128 sift-shaped f32, squared L2, M = 32, ef_construction = 100"}
    pts = datagen.sift_shaped(a.n, 128, 1)
    q = datagen.sift_shaped(a.nq, 128, 2)
    t0 = time.time()
    ix, _ = abi.Index.build(pts, M=32, ef_construction=100, seed=1)
    res["build_s"] = round(time.time() - t0, 1)
    del pts
    d_q = torch.from_numpy(q).cuda()
    d1000 = exact_k(torch, ix, d_q, a.nq, max(RANKS))
    radii = [float(np.median(d1000[:, r - 1])) for r in RANKS]
    del d1000
    res["exact"], res["graph"] = [], []
    e_off, e_ids, e_dist = {}, {}, {}
    for rank, radius in zip(RANKS, radii):
        off, ids, dist, ms = timed(torch, abi, lambda cap, o, i, d: ix.range_search_device(d_q.data_ptr(), a.nq, radius, cap, o, i, d),
                                   a.nq, a.reps)
        e_off[radius], e_ids[radius], e_dist[radius] = off, ids, dist
        counts = np.diff(off)
        r = {"neighbour_rank": rank, "radius": radius, "ms_per_call": median(ms), "ms_all": ms,
             "hits_per_query_mean": float(counts.mean()), "hits_per_query_max": int(counts.max())}
        res["exact"].append(r)
        print(json.dumps({"exact": r}), flush=True)
    runs = {}
    for ef in EFS:
        for (rank, radius), ex in zip(zip(RANKS, radii), res["exact"]):
            off, ids, dist, ms = timed(torch, abi, lambda cap, o, i, d: ix.graph_range_search_device(d_q.data_ptr(), a.nq, radius, cap, o, i,
                                                                                                 d, ef_search=ef), a.nq, a.reps)
            counts = np.diff(off)
            r = {"ef_search": ef, "neighbour_rank": rank, "radius": radius, "ms_per_call": median(ms), "ms_all": ms,
                 "exact_ms_per_call": ex["ms_per_call"], "speedup_vs_exact": ex["ms_per_call"] / median(ms),
                 "hits_per_query_mean": float(counts.mean()), "hits_per_query_max": int(counts.max()),
                 "recall_vs_exact": recall(off, ids, e_off[radius], e_ids[radius]),
                 "subset_of_exact": is_subset(off, ids, e_off[radius], e_ids[radius], a.nq)}
            res["graph"].append(r)
            runs[(ef, radius)] = (off, ids, dist)
            print(json.dumps({"graph": r}), flush=True)
    if a.check:
        stored, zero, upper = ix.export_graph()
        res["statement_check"] = check_against_statement(O, stored, zero, upper, 32, q[:a.check], runs, list(e_off.values()))
        print(json.dumps({"statement_check": res["statement_check"]}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k not in ("exact", "graph")}))


if __name__ == "__main__":
    main()
