"""Where one K1 expansion's time goes (DESIGN §5): builds a copy of the library with the phase clock on (-DIDB_K1_PHASES, into a
temporary directory; the product build has it off), runs the headline workload through it and prints one JSON line with each
phase's share of the warps' cycles and the cycles per expansion.

  python scripts/k1_phases.py [--lib PATH] [--n 1000000] [--dim 128] [--batch 10000] [--steps 5] [--ef 100] [--data sift|uniform]
  python scripts/k1_phases.py --sass LIB     static SASS instruction counts of the headline K1 instantiation in LIB (no GPU needed)

--lib: an instrumented library built beforehand (make -C instant-distance_b200/csrc EXTRA=-DIDB_K1_PHASES LIBDIR=... OBJDIR=...).
The tallies come from the CH = 1 kernels (rows of up to 128 elements), which hold the headline instantiation.
"""
import argparse
import collections
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "instant-distance_b200", "csrc")
HEADLINE = "_ZN3idb13search_kernelILi1ELi2ELi4ELi16ELi4ENS_6RowF32ELb1ELb0EEEvNS_10SearchArgsE"
# order of K1Phase in hnsw_device.cuh
PHASES = ["pop", "adjacency_load", "visited_probe_commit", "screen_loads", "screen_math", "gather_and_distances", "admission_merge", "ties"]
EVENTS = ["expansions", "screen_batches", "distance_batches", "distance_row_slots", "distance_rows"]


def sass_counts(lib):
    """Static instruction count of the headline instantiation, in total and by opcode."""
    out = subprocess.run(["cuobjdump", "-sass", "-fun", HEADLINE, lib], capture_output=True, text=True, check=True).stdout
    ops = collections.Counter()
    for line in out.splitlines():
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m:
            ops[m.group(1).split(".")[0]] += 1
    return {"function": HEADLINE, "instructions": sum(ops.values()), "by_opcode": dict(ops.most_common())}


def build_instrumented():
    tmp = tempfile.mkdtemp(prefix="idb_k1_phases_")
    jobs = str(max(1, min(8, os.cpu_count() or 1)))
    subprocess.check_call(["make", "-C", CSRC, "-j", jobs, "-s", "EXTRA=-DIDB_K1_PHASES", f"LIBDIR={tmp}/lib", f"OBJDIR={tmp}/obj"])
    return os.path.join(tmp, "lib", "libinstant_distance_b200.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--sass", metavar="LIB", default=None)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--ef", type=int, default=100)
    ap.add_argument("--M", type=int, default=32)
    ap.add_argument("--efc", type=int, default=100)
    ap.add_argument("--seed", type=int, default=20260923)
    ap.add_argument("--data", default="sift", choices=["sift", "uniform"])
    a = ap.parse_args()
    if a.sass:
        print(json.dumps(sass_counts(a.sass)), flush=True)
        return

    lib = a.lib or build_instrumented()
    os.environ["IDB_LIB_PATH"] = lib  # read when _abi is imported
    sys.path.insert(0, ROOT)
    import bench  # noqa: E402
    import torch  # noqa: E402

    from instant_distance_b200 import _abi  # noqa: E402

    L = ctypes.CDLL(lib)
    if not hasattr(L, "idb_debug_k1_phases"):
        raise SystemExit(f"{lib} was built without -DIDB_K1_PHASES")
    L.idb_debug_k1_phases.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    nslots = len(PHASES) + len(EVENTS)
    buf = (ctypes.c_ulonglong * nslots)()

    gen = bench.generator(a.data)
    pts = gen(a.n, a.dim, 1)
    p, zero, upper, _ = bench.obtain_graph(pts, a.n, a.dim, a.data, 1, a.M, a.efc, a.ef, a.seed, 0, use_abi=True)
    del pts
    qs = [torch.from_numpy(gen(a.batch, a.dim, 5000 + s)).cuda() for s in range(a.steps + 2)]
    ids = torch.empty((a.batch, 10), dtype=torch.int32, device="cuda")
    dist = torch.empty((a.batch, 10), dtype=torch.float32, device="cuda")
    lens = torch.empty((a.batch,), dtype=torch.int32, device="cuda")
    ix = _abi.Index.from_graph(p, zero, upper, a.M, a.ef)

    def step(q):
        ix.search_device(q.data_ptr(), a.batch, a.ef, 10, ids.data_ptr(), dist.data_ptr(), lens.data_ptr())
        ix.sync()

    for q in qs[:2]:
        step(q)
    if L.idb_debug_k1_phases(buf, 1) != nslots:  # drop the warm-up's (and the graph build's) tallies
        raise SystemExit("idb_debug_k1_phases failed")
    n_expand = 0
    for q in qs[2:]:
        step(q)
        c = ix.last_counters(a.batch)
        n_expand += int(c[:, 0].sum() + c[:, 2].sum())
    if L.idb_debug_k1_phases(buf, 1) != nslots:
        raise SystemExit("idb_debug_k1_phases failed")
    ix.close()
    v = list(buf)
    cyc = dict(zip(PHASES, v[:len(PHASES)]))
    ev = dict(zip(EVENTS, v[len(PHASES):]))
    total = sum(cyc.values())
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({
        "what": f"K1 phase clock (clock64 per warp, summed over warps), {a.n} x {a.dim} {a.data}, ef={a.ef}, {a.batch}-query batches, "
                f"{a.steps} batches after 2 warm-up batches",
        "gpu": gpu, "lib": os.path.basename(os.path.dirname(os.path.dirname(lib))),
        "expansions": ev["expansions"], "expansions_from_counters": n_expand,
        "cycles_per_expansion": total / max(1, ev["expansions"]),
        "phase_share": {k: x / max(1, total) for k, x in cyc.items()},
        "phase_cycles_per_expansion": {k: x / max(1, ev["expansions"]) for k, x in cyc.items()},
        "screen_batches_per_expansion": ev["screen_batches"] / max(1, ev["expansions"]),
        # batch_distances_impl: batches, row slots loaded and rows used (the slots past the rows are predicated off)
        "distance_batches_per_expansion": ev["distance_batches"] / max(1, ev["expansions"]),
        "distance_rows_per_expansion": ev["distance_rows"] / max(1, ev["expansions"]),
        "distance_row_slots_per_expansion": ev["distance_row_slots"] / max(1, ev["expansions"]),
        "distance_rows_per_slot": ev["distance_rows"] / max(1, ev["distance_row_slots"]),
    }), flush=True)


if __name__ == "__main__":
    main()
