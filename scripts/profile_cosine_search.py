"""A cosine index searched in 10k-query batches under torch.profiler: the device time of normalize_rows_kernel (the one launch a cosine
search adds: the queries' canonical normalisation, DESIGN §3a) next to K1's, per batch.  Prints one JSON line; --trace DIR also writes
the Chrome trace there.

  python scripts/profile_cosine_search.py [--n 1000000] [--dim 128] [--batch 10000] [--steps 10] [--trace DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "instant-distance_b200", "python"))
from instant_distance_b200 import _abi  # noqa: E402
from tests import datagen  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--ef", type=int, default=100)
    ap.add_argument("--trace", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    ix, _ = _abi.Index.build(datagen.sift_shaped(a.n, a.dim, 1), seed=20260923, metric="cosine")
    qs = [torch.from_numpy(datagen.sift_shaped(a.batch, a.dim, 5000 + s)).cuda() for s in range(a.steps + 3)]
    ids = torch.empty((a.batch, 10), dtype=torch.int32, device="cuda")
    dist = torch.empty((a.batch, 10), dtype=torch.float32, device="cuda")
    lens = torch.empty((a.batch,), dtype=torch.int32, device="cuda")

    def step(q):
        ix.search_device(q.data_ptr(), a.batch, a.ef, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr())
        ix.sync()

    for q in qs[:3]:
        step(q)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for q in qs[3:]:
            step(q)
    if a.trace:
        os.makedirs(a.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(a.trace, "cosine_search.pt.trace.json"))
    kernels = {}
    for e in prof.key_averages():
        for name in ("normalize_rows_kernel", "search_kernel"):
            if name in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                k = kernels.setdefault(name, {"launches": 0, "us_total": 0.0})
                k["launches"] += e.count
                k["us_total"] += t
    for k in kernels.values():
        k["us_per_batch"] = k["us_total"] / a.steps
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"what": f"cosine search, {a.n} x {a.dim} sift-shaped, ef={a.ef}, {a.batch}-query batches, {a.steps} batches under "
                              "torch.profiler (device time per kernel; search_kernel includes its normally idle retry launch)",
                      "gpu": gpu, "kernels": kernels}), flush=True)
    ix.close()


if __name__ == "__main__":
    main()
