"""Worker of tests/test_host_wide_groups_fake_runtime.py: GROUP BY over up to eight columns through the host executor over the
no-op runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory).
Prints one "WIDE {json}" line per run.  Not a test by itself.

    host_wide_groups_worker.py runs       TPC-H Q10, Q18, an 8-key plan and a numeric-key scan on both kernel routes, with and without a 16 KB budget
    host_wide_groups_worker.py refusal    a 9-key plan
    host_wide_groups_worker.py frees      every device allocation of Q18 and of the 8-key plan failing in turn"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import wide_groups as W  # noqa: E402
from cloudberry_b200 import capi, tpch_q10_q18 as Q  # noqa: E402


def emit(rec):
    print("WIDE " + json.dumps(rec), flush=True)


def plans():
    return (("q10", Q.q10_plan(sf=0.01)), ("q18", Q.q18_plan(threshold=250, sf=0.01)), ("keys8", W.plan(W.KEYS[:8])),
            ("num2", W.scan_plan(["k_num", "k_int4"])))


def run(ctx, ex, plan):
    """the run's code, rows, launches, and the kernel that filled the last aggregate table (the launch after its k_agg_init)"""
    before = ctx.launches()
    ctx.trace_begin()
    try:
        res = ex.run(plan)
        rec = {"rc": 0, "rows": len(res.rows)}
    except capi.CbgpuError as e:
        rec = {"rc": e.code, "msg": str(e)}
    names = [n for n, _ in ctx.trace_end()]
    inits = [i for i, n in enumerate(names) if n == "k_agg_init"]
    return dict(rec, launches=ctx.launches() - before, agg_inits=len(inits),
                agg_kernel=names[inits[-1] + 1] if inits and inits[-1] + 1 < len(names) else None)


def main():
    ctx = capi.Context(0)
    q = [capi.DeviceRelation.from_host(ctx, r) for r in Q.gen_tables(0.01, capi.hashbpchar)]
    w = [capi.DeviceRelation.from_host(ctx, r) for r in W.tables(2000, capi.hashbpchar, nulls=True)]
    if sys.argv[1] == "runs":
        for generic in (False, True):
            for mem_kb in (0, 16):
                exq, exw = (capi.Executor(ctx, d, force_generic=generic, operator_mem_kb=mem_kb) for d in (q, w))
                for name, plan in plans():
                    emit(dict(run(ctx, exw if name in ("keys8", "num2") else exq, plan), name=name, generic=generic, mem_kb=mem_kb))
                exq.close()
                exw.close()
    elif sys.argv[1] == "refusal":
        ex = capi.Executor(ctx, w)
        emit(dict(run(ctx, ex, W.plan(W.KEYS)), name="keys9"))
        ex.close()
    else:
        fake = C.CDLL(None)
        fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
        fake.fake_cudart_live_allocs.restype = C.c_long
        for name, plan in plans()[1:3]:
            ex = capi.Executor(ctx, w if name == "keys8" else q)
            k, codes, leaks = 0, [], []
            while True:
                k += 1
                base = fake.fake_cudart_live_allocs()
                fake.fake_cudart_fail_alloc_in(k)
                r = run(ctx, ex, plan)
                fake.fake_cudart_fail_alloc_in(0)
                if fake.fake_cudart_live_allocs() != base:
                    leaks.append([k, fake.fake_cudart_live_allocs() - base])
                if r["rc"] == 0:
                    break
                codes.append(r["rc"])
            emit(dict(name=name, failed=k - 1, codes=sorted(set(codes)), leaks=leaks, after=run(ctx, ex, plan)["rc"]))
            ex.close()
    for d in q + w:
        d.free()
    ctx.close()


if __name__ == "__main__":
    main()
