"""Time the two device top-N entry points on the same seeded relations (-m gpu machines only).

cbgpu_topn (LIMIT <= 64, integer keys without NULLs) and cbgpu_topn_select (any LIMIT, NULL and float8 keys) alternate at LIMIT
10 and 64 over synthetic relations of 10^6 and 10^8 rows - an int8 key of random values, then a Q3-like (revenue sum hi, lo)
pair whose hi is constant - and cbgpu_topn_select alone at LIMIT 100, 10^4 and 10^6.  Both answers are compared on every
input.  Each timing is the median of --reps calls, a host clock around the call (which ends in a device synchronise and the
indices' copy to the host; the Python list of indices is built inside it too), printed with the card's name and power limit
as one JSON line.

    python tools/topn_bench.py [--rows 1000000 100000000] [--reps 10]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402
from cloudberry_b200.relation import HostRelation  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def old_topn(ctx, dev, keys, limit):
    n = len(keys)
    A = C.c_int32 * n
    idx = (C.c_uint32 * 64)()
    nout = C.c_int64(0)
    ctx.check(ctx.L.cbgpu_topn(ctx.h, dev.h, A(*[k["col"] for k in keys]), A(*[k.get("descending", 0) for k in keys]),
                               A(*[k.get("unsigned_cmp", 0) for k in keys]), n, limit, idx, C.byref(nout)))
    return list(idx[:nout.value])


def timed(ctx, fn, reps):
    out, ms = None, []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()                                   # ends in a device synchronise (the indices' copy to the host)
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[10**6, 10**8])
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    ctx = capi.Context(0)
    gpu = card()
    rng = np.random.default_rng(42)
    for n in a.rows:
        cols = [rng.integers(-2**62, 2**62, n), np.zeros(n, dtype=np.int64), rng.integers(0, 2**40, n)]
        dev = capi.DeviceRelation.from_host(ctx, HostRelation("t", ["a", "hi", "lo"], [P.INT8] * 3, cols))
        del cols
        inputs = {"int8": [dict(col=0)], "sum_hi_lo_desc": [dict(col=1, descending=1), dict(col=2, unsigned_cmp=1, descending=1)]}
        for name, keys in inputs.items():
            for limit in (10, 64):
                timed(ctx, lambda: old_topn(ctx, dev, keys, limit), 2)
                timed(ctx, lambda: capi.topn_select(ctx, dev, keys, limit), 2)
                t_old, t_new = [], []
                for _ in range(a.reps):          # alternate the two entry points
                    want, ms = timed(ctx, lambda: old_topn(ctx, dev, keys, limit), 1)
                    t_old.append(ms)
                    got, ms = timed(ctx, lambda: capi.topn_select(ctx, dev, keys, limit), 1)
                    t_new.append(ms)
                    assert got == want, (n, name, limit)
                print(json.dumps({"gpu": gpu, "rows": n, "keys": name, "limit": limit, "cbgpu_topn_ms": round(statistics.median(t_old), 3),
                                  "cbgpu_topn_select_ms": round(statistics.median(t_new), 3)}), flush=True)
            for limit in (100, 10**4, 10**6):
                timed(ctx, lambda: capi.topn_select(ctx, dev, keys, limit), 1)
                _, ms = timed(ctx, lambda: capi.topn_select(ctx, dev, keys, limit), a.reps)
                print(json.dumps({"gpu": gpu, "rows": n, "keys": name, "limit": limit, "cbgpu_topn_select_ms": round(ms, 3)}), flush=True)
        dev.free()
    ctx.close()


if __name__ == "__main__":
    main()
