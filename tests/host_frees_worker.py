"""Worker of tests/test_host_frees_fake_runtime.py: makes every device allocation of a plan or of a library call fail in turn
over the no-op runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host
memory, and the runtime counts the device allocations still live).  Prints one JSON object.  Not a test by itself."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cloudberry_b200 import capi, ssb, tpch  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402

fake = C.CDLL(None)
fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
fake.fake_cudart_poison_int_d2h.argtypes = [C.c_long, C.c_int]
fake.fake_cudart_live_allocs.restype = C.c_long
fake.fake_cudart_device_allocs.restype = C.c_long
live = fake.fake_cudart_live_allocs
MAX_ALLOCS = 2000
NOMEM = -5


def sweep(attempt):
    """attempt(n) -> (code, extra): one run with the n-th device allocation failing (0: none), its arguments made and freed
    inside.  Returns the clean run's allocations, launches and what it left, then each failure's code and what it left."""
    ctx = sweep.ctx
    attempt(0)                                      # first use: what the context keeps for later calls (scratch grown on demand)
    base, a0, l0 = live(), fake.fake_cudart_device_allocs(), ctx.launches()
    code, _ = attempt(0)
    out = {"clean": {"code": code, "left": live() - base, "allocs": fake.fake_cudart_device_allocs() - a0,
                     "launches": ctx.launches() - l0},
           "failed": 0, "codes": [], "leaks": [], "bad_out": [], "not_alloc": []}
    for n in range(1, MAX_ALLOCS):
        base = live()
        code, extra = attempt(n)
        if code == 0:
            break
        out["failed"] += 1
        if code not in out["codes"]:
            out["codes"].append(code)
        if live() != base:
            out["leaks"].append([n, live() - base])
        if extra:
            out["bad_out"].append([n, extra])
        if code != NOMEM and "fake runtime error" not in ctx.error() + sweep.msg:
            out["not_alloc"].append([n, code, sweep.msg or ctx.error()])
        sweep.msg = ""
    return out


def failing(n, call):
    fake.fake_cudart_fail_alloc_in(n)
    try:
        return call()
    finally:
        fake.fake_cudart_fail_alloc_in(0)


def plan_sweep(make, plan):
    """make() -> an executor or cluster with run() and close(); the run after each failure, on the same object, must succeed"""
    def attempt(n):
        ex = make()
        try:
            failing(n, lambda: ex.run(plan))
            code, after = 0, None
        except capi.CbgpuError as e:
            code = e.code
            sweep.msg = str(e)      # a cluster reports a segment's error with code -1 and the segment's message
            try:
                ex.run(plan)
                after = None
            except capi.CbgpuError as e2:
                after = "next run: %d %s" % (e2.code, e2)
        ex.close()
        return code, after
    return sweep(attempt)


def main():
    out = {"plans": {}, "calls": {}}
    ctx = capi.Context(0)
    sweep.ctx = ctx
    sweep.msg = ""
    L = ctx.L
    rels, _ = tpch.load_golden(capi.hashbpchar)
    dev = [capi.DeviceRelation.from_host(ctx, r) for r in rels]
    seg = tpch.SEGMENTS.index("MACHINERY")
    reg = tpch.REGIONS.index("AMERICA")
    li, o = rels[0], rels[1]

    def executor(**kw):
        return lambda: capi.Executor(ctx, dev, **kw)

    def cluster():
        return lambda: capi.Cluster(ctx, [dev, dev, dev])

    plans = out["plans"]
    for generic in (False, True):
        for name, plan in (("q1", tpch.q1_plan(1)), ("q3", tpch.q3_plan(seg, 1)), ("q5", tpch.q5_plan(reg, 1))):
            plans[name + ("_generic" if generic else "")] = plan_sweep(executor(force_generic=generic), plan)
    plans["q5_16kb"] = plan_sweep(executor(operator_mem_kb=16), tpch.q5_plan(reg, 1))
    so = P.SeqScan(2, [("o_orderkey", P.Var(2, o.attno("o_orderkey"), P.INT8)), ("o_custkey", P.Var(2, o.attno("o_custkey"), P.INT4))])
    sl = P.SeqScan(1, [("l_orderkey", P.Var(1, li.attno("l_orderkey"), P.INT8)), ("l_suppkey", P.Var(1, li.attno("l_suppkey"), P.INT4))])

    def ol_join(jt):
        hh = P.Hash(so, [P.out_var(so, 1)])
        return P.HashJoin(jt, sl, hh, [P.out_var(sl, 1)], [("l_suppkey", P.out_var(sl, 2)), ("o_custkey", P.InnerVar(2, P.INT4))])
    jj = ol_join(P.JOIN_INNER)
    plans["orders_lineitem_16kb"] = plan_sweep(executor(operator_mem_kb=16), P.Agg(
        jj, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("l_suppkey", P.out_var(jj, 1)), ("n", P.Aggref(P.AGG_COUNT_STAR))], num_groups=64))
    for name, jt in (("right_join", P.JOIN_RIGHT), ("full_join", P.JOIN_FULL)):
        plans[name] = plan_sweep(executor(), P.Agg(ol_join(jt), P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR))]))
    sc = P.SeqScan(1, [(n, P.Var(1, li.attno(n), *li.var(n)[1:])) for n in ("l_returnflag", "l_quantity", "l_orderkey")])
    v = tpch._child_var(sc)
    keys_t = [("l_returnflag", v("l_returnflag")), ("s", P.Aggref(P.AGG_SUM, v("l_quantity")))]
    plans["having"] = plan_sweep(executor(), P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], keys_t, num_groups=8,
                                                   quals=[P.OpExpr(P.OP_GT, P.OuterVar(2, P.NUMERIC, 2), P.NumericConst("1"))]))
    plans["limit_sort_agg"] = plan_sweep(executor(), P.LimitSort(
        P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], keys_t, num_groups=8), [(1, False)], 2))
    plans["q3_3seg"] = plan_sweep(cluster(), tpch.q3_plan(seg, 3, customer_replicated=False))
    plans["q5_3seg"] = plan_sweep(cluster(), tpch.q5_plan(reg, 3, replicated=False))
    plans["q3_merge_gather_3seg"] = plan_sweep(cluster(), tpch.q3_plan(seg, 3, merge_gather=True))

    # Q3 with each 4-byte read-back in turn reporting a device error: an error, and nothing left behind
    de = {"raised": 0, "leaks": []}
    for n in range(1, 60):
        ex = capi.Executor(ctx, dev)
        base = live()
        fake.fake_cudart_poison_int_d2h(n, -6)
        try:
            ex.run(tpch.q3_plan(seg, 1))
            raised = False
        except capi.CbgpuError:
            raised = True
        fake.fake_cudart_poison_int_d2h(0, 0)
        ex.close()
        if live() != base:
            de["leaks"].append([n, live() - base])
        if not raised:
            break
        de["raised"] += 1
    out["status_word"] = de

    import host_batched_pairs_worker as BP
    import host_join_filter_worker as JF
    fo, do = BP.fact(20011), BP.dim(4000, 3)
    fdev = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
    for name, jt in (("left", P.JOIN_LEFT), ("semi", P.JOIN_SEMI), ("anti", P.JOIN_ANTI)):
        plans["join_filter_" + name] = plan_sweep(lambda: capi.Executor(ctx, fdev), JF.join(jt, fo, do))
    for d in fdev:
        d.free()
    srels = ssb.gen_tables(0.01, capi.hashbpchar)
    if srels is not None:
        sdev = [capi.DeviceRelation.from_host(ctx, r) for r in srels]
        plans["ssb_q4_1"] = plan_sweep(lambda: capi.Executor(ctx, sdev), ssb.q4_1_plan())
        for d in sdev:
            d.free()
    for d in dev:
        d.free()

    # ---- the library's calls one by one: arguments made before the failing call, freed after it ----
    calls = out["calls"]
    i32 = C.c_int32

    def rel(nrows, types, nulls_col=None):
        r = capi.DeviceRelation(ctx, nrows, types)
        if nulls_col is not None:
            w = P.TYPE_WIDTH[types[nulls_col]]
            ctx.check(L.cbgpu_rel_load_column(r.h, nulls_col, bytes(w * nrows), bytes(nrows)))
        return r

    def ctx_create(n):
        h = C.c_void_p()
        rc = failing(n, lambda: L.cbgpu_ctx_create(0, C.byref(h)))
        bad = rc != 0 and h.value is not None
        if rc == 0:
            L.cbgpu_ctx_destroy(h)
        return rc, bad
    calls["ctx_create"] = sweep(ctx_create)

    def rel_create(nrows, ncols):
        def attempt(n):
            h = C.c_void_p()
            rc = failing(n, lambda: L.cbgpu_rel_create(ctx.h, nrows, ncols, (i32 * ncols)(*[P.INT8] * ncols), None, C.byref(h)))
            bad = rc != 0 and h.value is not None
            if rc == 0:
                L.cbgpu_rel_free(h)
            return rc, bad
        return attempt
    calls["rel_create_slab"] = sweep(rel_create(1000, 6))
    calls["rel_create_per_column"] = sweep(rel_create(3 << 20, 3))        # 72 MB: one allocation per column

    def ht_build(nbatch):
        def attempt(n):
            inner = rel(4000, [P.INT4, P.INT8])
            h = C.c_void_p()
            rc = failing(n, lambda: L.cbgpu_ht_build(ctx.h, inner.h, (i32 * 1)(0), 1, nbatch, C.byref(h)))
            bad = rc != 0 and h.value is not None
            if rc == 0:
                L.cbgpu_ht_free(h)
            inner.free()
            return rc, bad
        return attempt
    calls["ht_build_1"] = sweep(ht_build(1))
    calls["ht_build_16"] = sweep(ht_build(16))

    L.cbgpu_agg_create.argtypes = [C.c_void_p, i32, i32, C.POINTER(i32), C.c_int64, C.POINTER(C.c_void_p)]
    L.cbgpu_agg_free.argtypes = [C.c_void_p]
    L.cbgpu_agg_free.restype = None
    L.cbgpu_agg_to_rel.argtypes = [C.c_void_p, C.POINTER(i32), C.POINTER(C.c_void_p)]

    def agg_create(n):
        h = C.c_void_p()
        rc = failing(n, lambda: L.cbgpu_agg_create(ctx.h, 2, 3, None, 1000, C.byref(h)))
        bad = rc != 0 and h.value is not None
        if rc == 0:
            L.cbgpu_agg_free(h)
        return rc, bad
    calls["agg_create"] = sweep(agg_create)

    def agg_to_rel(n):
        t = C.c_void_p()
        ctx.check(L.cbgpu_agg_create(ctx.h, 2, 3, None, 1000, C.byref(t)))
        h = C.c_void_p()
        rc = failing(n, lambda: L.cbgpu_agg_to_rel(t, (i32 * 2)(P.INT4, P.INT8), C.byref(h)))
        bad = rc != 0 and h.value is not None
        if rc == 0:
            L.cbgpu_rel_free(h)
        L.cbgpu_agg_free(t)
        return rc, bad
    calls["agg_to_rel"] = sweep(agg_to_rel)

    def dict_create(n):
        h = C.c_void_p()
        rc = failing(n, lambda: L.cbgpu_dict_create(ctx.h, 100, 4096, 1, C.byref(h)))
        bad = rc != 0 and h.value is not None
        if rc == 0:
            L.cbgpu_dict_free(h)
        return rc, bad
    calls["dict_create"] = sweep(dict_create)

    def topn(nrows):
        def attempt(n):
            r = rel(nrows, [P.INT8, P.INT8])
            idx, nout = (C.c_uint32 * 64)(), C.c_int64()
            one = (i32 * 2)(0, 1)
            rc = failing(n, lambda: L.cbgpu_topn(ctx.h, r.h, one, (i32 * 2)(1, 0), None, 2, 40, idx, C.byref(nout)))
            r.free()
            return rc, None
        return attempt
    calls["topn_4096"] = sweep(topn(4096))
    calls["topn_10000"] = sweep(topn(10000))

    def merge(n):
        r = rel(1000, [P.INT8])
        order, nruns = C.c_void_p(), i32()
        fake.fake_cudart_poison_int_d2h(1, 1)           # one run boundary found: the call goes on to place the rows
        rc = failing(n, lambda: L.cbgpu_merge_sorted_runs(ctx.h, r.h, (i32 * 1)(0), (i32 * 1)(0), None, 1, 4, C.byref(order),
                                                          C.byref(nruns)))
        fake.fake_cudart_poison_int_d2h(0, 0)
        bad = rc != 0 and order.value is not None
        if rc == 0:
            L.cbgpu_dev_free(ctx.h, order)
        r.free()
        return rc, bad
    calls["merge_sorted_runs"] = sweep(merge)

    L.cbgpu_rel_read_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]

    def read_rows(n):
        r = rel(1000, [P.INT8, P.INT4], nulls_col=1)
        idx = np.arange(0, 1000, 7, dtype=np.uint32)
        vals = np.zeros(len(idx) * 2, dtype=np.int64)
        nulls = np.zeros(len(idx) * 2, dtype=np.uint8)
        rc = failing(n, lambda: L.cbgpu_rel_read_rows(r.h, idx.ctypes.data, len(idx), vals.ctypes.data, nulls.ctypes.data))
        r.free()
        return rc, None
    calls["rel_read_rows"] = sweep(read_rows)

    def take_rows(n):
        src = rel(1000, [P.INT8, P.INT4], nulls_col=1)
        dst = rel(100, [P.INT8, P.INT4])
        d_idx = C.c_void_p()
        ctx.check(L.cbgpu_dev_alloc(ctx.h, 400, C.byref(d_idx)))
        rc = failing(n, lambda: L.cbgpu_rel_take_rows(dst.h, src.h, d_idx, 100))
        L.cbgpu_dev_free(ctx.h, d_idx)
        dst.free()
        src.free()
        return rc, None
    calls["rel_take_rows"] = sweep(take_rows)

    def load_narrow(n):
        r = rel(1000, [P.INT8])
        host = np.zeros(1000, dtype=np.int16)
        rc = failing(n, lambda: L.cbgpu_rel_load_column_narrow(r.h, 0, host.ctypes.data, 2))
        ctx.check(L.cbgpu_sync(ctx.h))
        r.free()
        return rc, None
    calls["rel_load_column_narrow"] = sweep(load_narrow)

    from test_aocs_format import CASES, TCASES, ZCASES, ZSTDCASES
    decode = {"int4": (P.INT4, 4, 0, 4), "int8": (P.INT8, 8, 0, 8), "date": (P.DATE, 4, 0, 4), "float8": (P.FLOAT8, 8, 0, 8),
              "bool": (P.BOOL, 1, 0, 1), "numeric": (P.NUMERIC, -1, 1, 4), "bpchar": (P.BPCHAR1, -1, 2, 4)}
    for kind, cases in ((0, CASES), (1, ZCASES), (2, ZSTDCASES)):
        for case in cases:
            name, typname, checksum, blocksize, dscale, nblocks, raw, values, nulls = case[:9]
            ctype, attlen, varkind, align = decode[typname]

            def aocs(n):
                r = capi.DeviceRelation(ctx, len(values) + 8, [ctype], dscales=[dscale])
                buf = np.frombuffer(raw, dtype=np.uint8)
                nr = C.c_int64()
                rc = failing(n, lambda: L.cbgpu_aocs_decode_column_ex(ctx.h, buf.ctypes.data, len(buf), 1 if checksum else 0, kind, attlen,
                                                                      varkind, align, r.h, 0, 0, C.byref(nr)))
                r.free()
                return rc, None
            calls["aocs_decode_%s" % name] = sweep(aocs)
    comp = {"": 0, "zlib": 1, "zstd": 2}
    for case in TCASES[:3]:
        name, typname, checksum, blocksize, nblocks, raw, values, nulls, cmp = case
        buf = np.frombuffer(raw, dtype=np.uint8)

        def collect(n):
            d = capi.DeviceDict(ctx, max_entries=8192, bpchar=typname == "bpchars")
            rc = failing(n, lambda: L.cbgpu_aocs_dict_collect(ctx.h, buf.ctypes.data, len(buf), 1 if checksum else 0, comp[cmp], 4, d.h))
            d.free()
            return rc, None

        def decode_dict(n):
            d = capi.DeviceDict(ctx, max_entries=8192, bpchar=typname == "bpchars")
            d.collect(raw, checksum, comp[cmp])
            d.finalize()
            r = capi.DeviceRelation(ctx, len(values), [P.DICT32])
            nr = C.c_int64()
            rc = failing(n, lambda: L.cbgpu_aocs_decode_dict_column(ctx.h, buf.ctypes.data, len(buf), 1 if checksum else 0, comp[cmp], 4,
                                                                    d.h, r.h, 0, 0, C.byref(nr)))
            r.free()
            d.free()
            return rc, None
        calls["aocs_dict_collect_%s" % name] = sweep(collect)
        calls["aocs_decode_dict_%s" % name] = sweep(decode_dict)

    a = {c[0]: c for c in CASES}["int4_plain"]

    def visimap(n):
        r = capi.DeviceRelation(ctx, len(a[7]) + 8, [P.INT4])
        entries = (capi.CbgpuVisimapEntry * 1)()
        payload = C.create_string_buffer(b"\x01\0\0\0\0\0", 6)
        entries[0].first_row_num = 0
        entries[0].data = C.cast(payload, C.c_void_p)
        entries[0].len = 6
        buf = np.frombuffer(a[6], dtype=np.uint8)
        nh = C.c_int64()
        rc = failing(n, lambda: L.cbgpu_aocs_apply_visimap(ctx.h, buf.ctypes.data, len(buf), 1 if a[2] else 0, entries, 1, r.h, 0,
                                                           C.byref(nh)))
        r.free()
        return rc, None
    calls["aocs_apply_visimap"] = sweep(visimap)

    ctx.close()
    print("HOSTFREES " + json.dumps(out))


if __name__ == "__main__":
    main()
