"""K1 on the headline workload under torch.profiler, with the screening pass off and on (DESIGN §4, §5): device time of
search_kernel per 10k-query batch, and the share of distance evaluations whose row was fetched in full.  Prints one JSON line.

  python scripts/profile_screen.py [--n 1000000] [--dim 128] [--batch 10000] [--steps 10] [--ef 100] [--data sift|uniform]
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
    ap.add_argument("--data", default="sift", choices=["sift", "uniform"])
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    make = datagen.sift_shaped if a.data == "sift" else datagen.uniform
    built, _ = _abi.Index.build(make(a.n, a.dim, 1), seed=20260923)
    g = built.export_graph()
    built.close()
    qs = [torch.from_numpy(make(a.batch, a.dim, 5000 + s)).cuda() for s in range(a.steps + 3)]
    ids = torch.empty((a.batch, 10), dtype=torch.int32, device="cuda")
    dist = torch.empty((a.batch, 10), dtype=torch.float32, device="cuda")
    lens = torch.empty((a.batch,), dtype=torch.int32, device="cuda")
    out = {}
    for screen in ("0", "1"):
        os.environ["IDB_SCREEN"] = screen  # read when the index is created
        ix = _abi.Index.from_graph(g[0], g[1], g[2], 32)

        def step(q):
            ix.search_device(q.data_ptr(), a.batch, a.ef, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr())
            ix.sync()

        for q in qs[:3]:
            step(q)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for q in qs[3:]:
                step(q)
        us = sum((getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
                 for e in prof.key_averages() if "search_kernel" in e.key)
        r = {"search_kernel_ms_per_batch": us / a.steps / 1000.0}
        if hasattr(ix, "last_full_fetches"):
            step(qs[-1])
            c = ix.last_counters(a.batch)
            n_dist = int(c[:, 1].sum() + c[:, 3].sum())
            r["full_fetch_share"] = ix.last_full_fetches(0) / n_dist
            r["distances_per_query"] = n_dist / a.batch
        out["screen_" + screen] = r
        ix.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"what": f"K1 (search_kernel incl. its idle retry launch), {a.n} x {a.dim} {a.data}, ef={a.ef}, {a.batch}-query "
                              f"batches, {a.steps} batches under torch.profiler", "gpu": gpu, **out}), flush=True)


if __name__ == "__main__":
    main()
