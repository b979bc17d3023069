#!/usr/bin/env python3
"""TPC-H Q21 (tpch_q21.q21_plan) on one GPU: wall time with no operator memory budget and with budgets that give the requested
batch counts for the largest build side (all of lineitem, under the semi join), each run's rows checked against the unbudgeted
run's.  Prints one JSON line: the GPU (name, power limit), per budget the largest nbatch used, the wall time of each run (host
clock around a query that ends in a read-back) and whether its rows equal the unbudgeted run's; then, from a separate
torch.profiler run per budget, the summed device time of the table fills, the filtered pair probes, the batch partition, the
prefix scans and the pipeline kernels (the scans of lineitem, orders, supplier and nation and the joins fused into them).

The tables are built on the host from tpch_q21's formulas (a few GB of host memory at SF10).

    python tools/q21_bench.py --sf 10 --batches 8 64 --reps 3 [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cloudberry_b200 import capi, tpch, tpch_q21  # noqa: E402

GROUPS = {"fill": ("k_ht_clear", "k_ht_build", "k_ht_batch_histogram"), "filtered_probe": ("k_ht_probe_filtered",),
          "partition": ("k_ht_partition_count", "k_ht_partition_write"), "prefix_scan": ("k_exclusive_scan_u64",),
          "pipelines": ("k_pipeline_generic", "k_probe_chain", "k_prefilter", "k_scan_agg")}


def budget_kb(G, rows, nbatch):
    """the smallest budget (KB) whose batch choice (cb_exec.c hash_build) is nbatch"""
    return 0 if nbatch <= 1 else -(-G.cbgpu_ht_bytes_for(-(-rows // nbatch)) // 1024)


def kernel_times(run):
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        return None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in GROUPS}
    total = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        total += us / 1000.0
        for k, names in GROUPS.items():
            if any(e.key.startswith(n) or ("%s<" % n) in e.key or ("%s(" % n) in e.key for n in names):
                out[k] += us / 1000.0
    out["all_device"] = total
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON line (nothing is written otherwise)")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines() if shutil.which("nvidia-smi") else []
    ctx = capi.Context(0)
    G = ctx.L
    G.cbgpu_ht_bytes_for.restype = C.c_int64
    G.cbgpu_ht_bytes_for.argtypes = [C.c_int64]
    t0 = time.perf_counter()
    host = tpch_q21.gen_tables(a.sf, capi.hashbpchar)
    rels = [capi.DeviceRelation.from_host(ctx, r) for r in host]
    del host
    nli = tpch.sizes(a.sf)["lineitem"]
    q = tpch_q21.q21_plan(limit=100)                       # the query's own LIMIT
    result = {"gpu": gpu[0] if gpu else None, "sf": a.sf, "lineitem": nli, "load_s": round(time.perf_counter() - t0, 1), "runs": []}
    base_rows = None
    for nb in [1] + a.batches:
        ex = capi.Executor(ctx, rels, operator_mem_kb=budget_kb(G, nli, nb))
        res = ex.run(q)                                    # warm-up
        used = max(v["hashjoin_nbatch"] for v in res.instrument.values())
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rows = ex.run(q).rows
            walls.append(round((time.perf_counter() - t0) * 1000.0, 2))
        base_rows = rows if base_rows is None else base_rows
        result["runs"].append({"nbatch": int(used), "budget_kb": budget_kb(G, nli, nb), "wall_ms": walls,
                               "rows_equal_unbudgeted": rows == base_rows, "nrows": len(rows),
                               "kernel_ms": kernel_times(lambda: ex.run(q))})
        ex.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "q21_bench.json"), "w") as f:
            f.write(line + "\n")
    for r in rels:
        r.free()
    ctx.close()


if __name__ == "__main__":
    main()
