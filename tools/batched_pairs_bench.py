#!/usr/bin/env python3
"""Cost of splitting a pair join's build side into batches: TPC-H orders probe Hash(lineitem) on l_orderkey (N:M, 1-7 lines
per order), aggregated, with no operator memory budget and with budgets that give the requested batch counts.  Prints one
JSON line: the GPU (name, power limit), per budget the batches used, the wall time of each run (host clock around a query
that ends in a read-back) and whether its rows equal the unbudgeted run's; then, from a separate torch.profiler run per
budget, the summed device time of the partition kernels, the pair count / write kernels, and the table fills.

    python tools/batched_pairs_bench.py --sf 10 --batches 8 64 --reps 3 [--out DIR]"""
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

from cloudberry_b200 import capi, harness, tpch  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402

GROUPS = {"partition": ("k_ht_partition_count", "k_ht_partition_write"), "pairs": ("k_ht_probe_pairs",),
          "scan": ("k_exclusive_scan_u64",), "fill": ("k_ht_clear", "k_ht_build")}


def plan():
    so = tpch._scan("orders", ["o_orderkey", "o_orderdate"])
    sl = tpch._scan("lineitem", ["l_orderkey", "l_quantity", "l_extendedprice"])
    h = P.Hash(sl, [P.out_var(sl, 1)])
    j = P.HashJoin(P.JOIN_INNER, so, h, [P.out_var(so, 1)],
                   [("o_orderdate", P.out_var(so, 2)), ("l_quantity", P.InnerVar(2, *P.out_type(sl, 2))),
                    ("l_extendedprice", P.InnerVar(3, *P.out_type(sl, 3)))])
    v = tpch._child_var(j)
    return P.Agg(j, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR)), ("sq", P.Aggref(P.AGG_SUM, v("l_quantity"))),
                                                        ("se", P.Aggref(P.AGG_SUM, v("l_extendedprice"))),
                                                        ("mx", P.Aggref(P.AGG_MAX, v("o_orderdate")))])


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
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        us = e.cuda_time_total if us is None else us
        for k, names in GROUPS.items():
            if e.key.startswith(names) or any(("%s<" % n) in e.key or ("%s(" % n) in e.key for n in names):
                out[k] += us / 1000.0
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
    rels, sz = harness.device_tables(ctx, a.sf)
    q = plan()
    result = {"gpu": gpu[0] if gpu else None, "sf": a.sf, "orders": sz["orders"], "lineitem": sz["lineitem"], "runs": []}
    base_rows = None
    for nb in [1] + a.batches:
        ex = capi.Executor(ctx, rels, operator_mem_kb=budget_kb(G, sz["lineitem"], nb))
        res = ex.run(q)                                    # warm-up
        used = max(v["hashjoin_nbatch"] for v in res.instrument.values())
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rows = ex.run(q).rows
            walls.append(round((time.perf_counter() - t0) * 1000.0, 2))
        base_rows = rows if base_rows is None else base_rows
        result["runs"].append({"nbatch": int(used), "budget_kb": budget_kb(G, sz["lineitem"], nb), "wall_ms": walls,
                               "rows_equal_unbudgeted": rows == base_rows, "rows": rows, "kernel_ms": kernel_times(lambda: ex.run(q))})
        ex.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "batched_pairs_bench.json"), "w") as f:
            f.write(line + "\n")
    for r in rels:
        r.free()
    ctx.close()


if __name__ == "__main__":
    main()
