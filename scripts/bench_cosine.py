"""The headline search workload under cosine distance (DESIGN §3a), next to the same workload under squared L2 in the same run.

1M x 128 sift-shaped points, M=32, ef_construction=100, ef_search=100 (raised until recall@10 >= 0.95), 10k-query batches issued
alternately on two submission lanes with queries and outputs resident in HBM — bench.py's device-resident protocol — for a cosine
index and a squared-L2 index built from the same rows, measured alternately (`--reps` times each).  Also: cosine recall@10 against
cosine brute force, and the GPU's ids, distance bytes, lengths and per-layer counters of one batch against the CPU statement of
cosine (tests/cosine_ref.py: the oracle's canonical squared L2 on the normalised rows, distances halved) on the same graph.
Prints one JSON line, with the card's name and power limit.

  python scripts/bench_cosine.py [--n 1000000] [--dim 128] [--steps 20] [--warmup 3] [--reps 2] [--parity-sample 10000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (bench.py's helpers: brute force, recall, host threads; its sys.path set-up)
from instant_distance_b200 import _abi  # noqa: E402
from tests import cosine_ref, datagen  # noqa: E402

K = bench.K


def device_qps(ix, dq, ef, steps, warmup, lanes=2):
    """bench.py's device-resident arm: `warmup` untimed batches, then `steps` batches round-robin over `lanes` lanes, device time."""
    import torch

    nq = dq[0].shape[0]
    outs = [(torch.empty((nq, K), dtype=torch.int32, device="cuda"), torch.empty((nq, K), dtype=torch.float32, device="cuda"),
             torch.empty((nq,), dtype=torch.int32, device="cuda")) for _ in range(lanes)]
    streams = [torch.cuda.ExternalStream(ix.lane_stream(l)) for l in range(lanes)]

    def step(s, lane):
        i, d, n = outs[lane]
        ix.search_device(dq[s].data_ptr(), nq, ef, K, i.data_ptr(), d.data_ptr(), n.data_ptr(), lane=lane)

    for s in range(warmup):
        step(s, s % lanes)
    ix.sync()
    torch.cuda.synchronize()
    ev0 = torch.cuda.Event(enable_timing=True)
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(lanes)]
    ev0.record(streams[0])
    for l in range(1, lanes):
        streams[l].wait_event(ev0)
    for s in range(warmup, warmup + steps):
        step(s, s % lanes)
    for l in range(lanes):
        ends[l].record(streams[l])
    torch.cuda.synchronize()
    ms = max(ev0.elapsed_time(e) for e in ends)
    assert ix.last_failures(0) == 0 and ix.last_failures(1) == 0
    return nq * steps / (ms / 1e3), ms / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--M", type=int, default=32)
    ap.add_argument("--efc", type=int, default=100)
    ap.add_argument("--ef", type=int, default=100)
    ap.add_argument("--seed", type=int, default=20260923)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--parity-sample", type=int, default=10_000)
    a = ap.parse_args()
    import torch

    from oracle import oracle as O

    pts = datagen.sift_shaped(a.n, a.dim, 1)
    kw = dict(M=a.M, ef_construction=a.efc, ef_search=a.ef, seed=a.seed)
    cos, _ = _abi.Index.build(pts, metric="cosine", **kw)
    l2, _ = _abi.Index.build(pts, **kw)
    del pts
    p, zero, upper = cos.export_graph()  # the normalised rows, PointId order

    rq = datagen.sift_shaped(1000, a.dim, 999)
    truth, _ = bench.brute_force_topk_torch(torch.from_numpy(p).cuda(), _abi.normalize(rq), K)  # L2 order on unit rows = cosine order
    torch.cuda.empty_cache()
    ef, recall = a.ef, 0.0
    for cand in [a.ef, 128, 160, 200, 256, 320, 400, 512, 768, 1024]:
        if cand < a.ef:
            continue
        ids, _, _ = cos.search(rq, ef_search=cand, k=K)
        ef, recall = cand, bench.recall_at_k(ids, truth)
        if recall >= 0.95:
            break

    host_q = [datagen.sift_shaped(a.batch, a.dim, 5000 + s) for s in range(a.warmup + a.steps)]
    dq = [torch.from_numpy(q).cuda() for q in host_q]
    runs = {"cosine": [], "l2sq": []}
    for _ in range(a.reps):
        for name, ix in (("l2sq", l2), ("cosine", cos)):
            runs[name].append(device_qps(ix, dq, ef, a.steps, a.warmup))

    T = bench.host_threads()
    sample = host_q[-1][:a.parity_sample]
    ox = O.from_graph(O.Graph(p, zero, upper, a.M, ef))
    o_ids, o_dist, o_len, o_cnt = cosine_ref.search(O, ox, sample, ef_search=ef, k=K, threads=T, counters=True)
    g_ids, g_dist, g_len = cos.search(sample, ef_search=ef, k=K)
    parity = bool((g_ids == o_ids).all() and g_dist.tobytes() == o_dist.tobytes() and (g_len == o_len).all()
                  and (cos.last_counters(len(sample)) == o_cnt).all())

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({
        "what": f"{a.n} x {a.dim} sift-shaped, M={a.M}, ef_construction={a.efc}, ef_search={ef}, batch={a.batch}, k={K}: device-resident "
                f"batches over two lanes, {a.warmup} warm + {a.steps} timed steps, cosine and squared-L2 indexes of the same rows measured "
                f"alternately {a.reps}x",
        "gpu": gpu, "cosine_qps": [r[0] for r in runs["cosine"]], "l2sq_qps": [r[0] for r in runs["l2sq"]],
        "cosine_ms_per_step": [r[1] for r in runs["cosine"]], "l2sq_ms_per_step": [r[1] for r in runs["l2sq"]],
        "cosine_recall_at_10": recall, "ef_search": ef,
        "parity_with_cpu_statement": parity, "parity_sample": len(sample)}), flush=True)
    cos.close()
    l2.close()


if __name__ == "__main__":
    main()
