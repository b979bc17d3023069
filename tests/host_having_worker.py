"""Worker of tests/test_host_having_fake_runtime.py: HAVING through the host executor and cbgpu_having_select over the no-op
runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory).
Prints one "HAVING {json}" line per run.  Not a test by itself.

    host_having_worker.py runs       Q18 and the HAVING shapes of test_gpu_capacity::test_having on both kernel routes, with
                                     and without a 16 KB budget; cbgpu_having_select over a relation of 1000 groups
    host_having_worker.py refusals   every HAVING shape the device path does not evaluate
    host_having_worker.py frees      every device allocation of cbgpu_having_select failing in turn"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cloudberry_b200 import capi, tpch_q10_q18 as Q  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402
from cloudberry_b200.relation import HostRelation  # noqa: E402

HAVING_OPS = [(capi.CBP_STATE, 1, capi.CBH_SUM | 2 << 8), (capi.CBP_CONST, 0, 300), (capi.CBP_GT, 0, 0)]


def emit(rec):
    print("HAVING " + json.dumps(rec), flush=True)


def lineitem_agg(rels, quals, keys=("l_orderkey",)):
    li = rels[0]
    sc = P.SeqScan(1, [(n, P.Var(1, li.attno(n), *li.var(n)[1:])) for n in ("l_orderkey", "l_quantity", "l_extendedprice")])
    v = lambda n: P.out_var(sc, ("l_orderkey", "l_quantity", "l_extendedprice").index(n) + 1)     # noqa: E731
    targets = [("l_orderkey", v("l_orderkey")), ("s", P.Aggref(P.AGG_SUM, v("l_quantity")))]
    return P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], targets, num_groups=1000, quals=[q(v) for q in quals])


def plans(rels):
    return [
        ("q18", Q.q18_plan(threshold=250, sf=0.01)),
        ("sum", lineitem_agg(rels, [lambda v: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_SUM, v("l_quantity")), P.NumericConst("250"))])),
        ("avg_count", lineitem_agg(rels, [
            lambda v: P.OpExpr(P.OP_LE, P.Aggref(P.AGG_AVG, v("l_extendedprice")), P.NumericConst("20000.50")),
            lambda v: P.OpExpr(P.OP_GE, P.Aggref(P.AGG_COUNT_STAR), P.Const(P.INT8, 5))])),
        ("bool", lineitem_agg(rels, [lambda v: P.BoolExpr(
            P.OR_EXPR, P.OpExpr(P.OP_EQ, P.Aggref(P.AGG_COUNT_STAR), P.Const(P.INT8, 7)),
            P.BoolExpr(P.NOT_EXPR, P.OpExpr(P.OP_GT, v("l_orderkey"), P.Const(P.INT8, 1000))))])),
    ]


def refusals(rels):
    s = lambda v: P.Aggref(P.AGG_SUM, v("l_quantity"))     # noqa: E731
    cust = rels[2]
    sc = P.SeqScan(3, [("c_name", P.Var(3, cust.attno("c_name"), *cust.var("c_name")[1:]))])
    dict_key = P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("c_name", P.out_var(sc, 1))], num_groups=100,
                     quals=[P.OpExpr(P.OP_EQ, P.out_var(sc, 1), P.Const(P.DICT32, 0))])
    return [
        ("arithmetic", lineitem_agg(rels, [lambda v: P.OpExpr(P.OP_GT, P.OpExpr(P.OP_ADD, s(v), s(v)), P.NumericConst("1"))]),
         "HAVING on the GPU path takes no arithmetic"),
        ("mixed", lineitem_agg(rels, [lambda v: P.OpExpr(P.OP_GT, s(v), P.Const(P.FLOAT8, 1.0))]),
         "compares two exact or two float8 values, not one of each"),
        ("text", lineitem_agg(rels, [lambda v: P.OpExpr(P.OP_EQ, v("l_orderkey"), P.TextConst("x"))]),
         "LIKE and IN lists of strings are only taken in the quals of a scan"),
        ("dict_key", dict_key, "HAVING on the GPU path compares no dictionary-coded grouping column"),
        ("in_list", lineitem_agg(rels, [lambda v: P.InList(v("l_orderkey"), [1, 2, 3])]),
         "HAVING on the GPU path takes no IN / ANY / ALL lists"),
        ("nine_aggs", lineitem_agg(rels, [lambda v, i=i: P.OpExpr(P.OP_GT, s(v), P.NumericConst(str(i))) for i in range(9)]),
         "more than 8 aggregates in HAVING"),
    ]


def run(ctx, ex, plan):
    before = ctx.launches()
    ctx.trace_begin()
    try:
        res = ex.run(plan)
        rec = {"rc": 0, "rows": len(res.rows)}
    except capi.CbgpuError as e:
        rec = {"rc": e.code, "msg": str(e)}
    names = [n for n, _ in ctx.trace_end()]
    return dict(rec, launches=ctx.launches() - before, having=[n for n in names if n.startswith("k_having")])


def groups(ctx, n):
    """a groups relation of n groups: an int8 key, one accumulator's (N, lo, hi)"""
    import numpy as np
    z = np.zeros(n, np.int64)
    return capi.DeviceRelation.from_host(ctx, HostRelation("g", ["k", "n", "lo", "hi"], [P.INT8] * 4, [z, z, z, z]))


def select(ctx, rel):
    before = ctx.launches()
    ctx.trace_begin()
    try:
        rec = {"rc": 0, "nsel": len(capi.having_select(ctx, rel, HAVING_OPS, 1))}
    except capi.CbgpuError as e:
        rec = {"rc": e.code, "msg": str(e)}
    return dict(rec, launches=ctx.launches() - before, having=[n for n, _ in ctx.trace_end()])


def main():
    ctx = capi.Context(0)
    rels = Q.gen_tables(0.01, capi.hashbpchar)
    dev = [capi.DeviceRelation.from_host(ctx, r) for r in rels]
    if sys.argv[1] == "runs":
        for generic in (False, True):
            for mem_kb in (0, 16):
                ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
                for name, plan in plans(rels):
                    emit(dict(run(ctx, ex, plan), name=name, generic=generic, mem_kb=mem_kb))
                ex.close()
        g = groups(ctx, 1000)
        emit(dict(select(ctx, g), name="entry_point"))
        g.free()
    elif sys.argv[1] == "refusals":
        ex = capi.Executor(ctx, dev)
        for name, plan, msg in refusals(rels):
            emit(dict(run(ctx, ex, plan), name=name, want=msg))
        ex.close()
    else:
        fake = C.CDLL(None)
        fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
        fake.fake_cudart_live_allocs.restype = C.c_long
        g = groups(ctx, 1000)
        k, codes, leaks = 0, [], []
        while True:
            k += 1
            base = fake.fake_cudart_live_allocs()
            fake.fake_cudart_fail_alloc_in(k)
            r = select(ctx, g)
            fake.fake_cudart_fail_alloc_in(0)
            if fake.fake_cudart_live_allocs() != base:
                leaks.append([k, fake.fake_cudart_live_allocs() - base])
            if r["rc"] == 0:
                break
            codes.append(r["rc"])
        emit(dict(name="entry_point", failed=k - 1, codes=sorted(set(codes)), leaks=leaks, after=select(ctx, g)["rc"]))
        g.free()
    for d in dev:
        d.free()
    ctx.close()


if __name__ == "__main__":
    main()
