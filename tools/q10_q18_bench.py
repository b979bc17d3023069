#!/usr/bin/env python3
"""TPC-H Q10 and Q18 (tpch_q10_q18) on one GPU.  Prints one JSON line: the GPU (name, power limit), and per query the wall time
of each run (host clock around a query that ends in a read-back) with the summed device time of its pipeline kernels
(instrument device_ms).  For Q18 it also reports the host HAVING step of its IN subquery (instrument having_ms: the host
reads every group's key and state, selects the groups that pass and uploads the selection), which is part of the wall time.
With --check-sf (default 1) both queries are run once more at that scale factor and their rows compared with the numpy
answers (result_check).

The tables are built on the host from tpch_q10_q18's formulas (a few GB of host memory at SF10).

    python tools/q10_q18_bench.py --sf 10 --reps 3 [--check-sf 1] [--threshold 300]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cloudberry_b200 import capi, tpch_q10_q18 as Q  # noqa: E402


def timed(ctx, ex, make_plan):
    ctx.sync()
    t = time.perf_counter()
    res = ex.run(make_plan())
    ms = (time.perf_counter() - t) * 1e3
    ins = res.instrument.values()
    return ms, sum(v["device_ms"] for v in ins), sum(v["having_ms"] for v in ins), len(res.rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threshold", type=int, default=300)
    ap.add_argument("--check-sf", type=float, default=1)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines() if shutil.which("nvidia-smi") else []
    ctx = capi.Context(0)
    out = {"gpu": gpu[0] if gpu else "not found", "sf": a.sf, "threshold": a.threshold}
    sf = int(a.sf) if a.sf == int(a.sf) else a.sf
    dev = [capi.DeviceRelation.from_host(ctx, r) for r in Q.gen_tables(sf, capi.hashbpchar)]
    ex = capi.Executor(ctx, dev)
    print("tables on the device", file=sys.stderr, flush=True)
    for name, make in (("q10", lambda: Q.q10_plan(sf=sf)), ("q18", lambda: Q.q18_plan(threshold=a.threshold, sf=sf))):
        timed(ctx, ex, make)                        # warm-up: module load, first allocations
        runs = [timed(ctx, ex, make) for _ in range(a.reps)]
        print(name, [round(r[0], 2) for r in runs], file=sys.stderr, flush=True)
        out[name] = {"wall_ms": [round(r[0], 2) for r in runs], "device_ms": [round(r[1], 2) for r in runs],
                     "rows": runs[0][3]}
        if name == "q18":
            out[name]["having_host_ms"] = [round(r[2], 2) for r in runs]
    ex.close()
    for d in dev:
        d.free()
    if a.check_sf:
        csf = int(a.check_sf) if a.check_sf == int(a.check_sf) else a.check_sf
        dev = [capi.DeviceRelation.from_host(ctx, r) for r in Q.gen_tables(csf, capi.hashbpchar)]
        ex = capi.Executor(ctx, dev)
        out["result_check"] = {"sf": a.check_sf,
                               "q10": [tuple(r) for r in ex.run(Q.q10_plan(sf=csf)).rows] == Q.q10_numpy_answer(csf),
                               "q18": [tuple(r) for r in ex.run(Q.q18_plan(threshold=a.threshold, sf=csf)).rows] ==
                               Q.q18_numpy_answer(csf, threshold=a.threshold)}
        ex.close()
        for d in dev:
            d.free()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
