"""Worker of tests/test_host_logic_fake_runtime.py: drives the host executor over the no-op runtime of tests/fake_runtime.py
(LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory).  Prints one JSON object.  Not a test by
itself."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cloudberry_b200 import capi, ssb, tpch  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402


def main():
    out = {"ran": {}, "refused": {}}
    G = capi.gpu()
    assert G.cbgpu_device_count() == 1
    ctx = capi.Context(0)
    rels, _ = tpch.load_golden(capi.hashbpchar)
    dev = [capi.DeviceRelation.from_host(ctx, r) for r in rels]
    seg = tpch.SEGMENTS.index("MACHINERY")
    reg = tpch.REGIONS.index("AMERICA")

    # 1. every plan shape of the metric goes through translation, program emission, kernel matching, launch and read-back
    for generic in (False, True):
        ex = capi.Executor(ctx, dev, force_generic=generic)
        for name, plan in (("q1", tpch.q1_plan(1)), ("q3", tpch.q3_plan(seg, 1)), ("q5", tpch.q5_plan(reg, 1))):
            before = ctx.launches()
            res = ex.run(plan)
            out["ran"]["%s%s" % (name, "_generic" if generic else "")] = {"rows": len(res.rows), "launches": ctx.launches() - before}
        ex.close()

    # 2. plans with Motions on a 3-segment cluster in one process (two-stage aggregation, redistributed joins)
    cl = capi.Cluster(ctx, [dev, dev, dev])
    for name, plan in (("q1_3seg", tpch.q1_plan(3)), ("q3_3seg", tpch.q3_plan(seg, 3, customer_replicated=False)),
                       ("q5_3seg", tpch.q5_plan(reg, 3, replicated=False))):
        before = ctx.launches()
        res = cl.run(plan)
        out["ran"][name] = {"rows": len(res.rows), "launches": ctx.launches() - before}
    cl.close()

    # 3. what the host must refuse, loudly and before any kernel: (plan builder, expected message fragment)
    li = rels[0]
    sc = P.SeqScan(1, [(n, P.Var(1, li.attno(n), *li.var(n)[1:])) for n in ("l_returnflag", "l_quantity", "l_orderkey")])
    v = tpch._child_var(sc)
    keys_t = [("l_returnflag", v("l_returnflag")), ("s", P.Aggref(P.AGG_SUM, v("l_quantity")))]

    def having():
        return P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], keys_t, num_groups=8,
                     quals=[P.OpExpr(P.OP_GT, P.OuterVar(2, P.NUMERIC, 2), P.NumericConst("1"))])

    def sorted_agg():
        return P.Agg(sc, P.AGG_SORTED, P.AGGSPLIT_SIMPLE, [1], keys_t, num_groups=8)

    def sort_without_limit():
        a = P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], keys_t, num_groups=8)
        return P.LimitSort(a, [(1, False)], -1)

    def right_join():
        o = rels[1]
        so = P.SeqScan(2, [("o_orderkey", P.Var(2, o.attno("o_orderkey"), P.INT8))])
        h = P.Hash(so, [P.out_var(so, 1)])
        # RIGHT joins run (pairs with a missing side); extra join quals on an outer join are still refused
        j = P.HashJoin(P.JOIN_RIGHT, sc, h, [P.out_var(sc, 3)], [("l_quantity", P.out_var(sc, 2))],
                       joinquals=[P.OpExpr(P.OP_GT, P.out_var(sc, 3), P.Const(P.INT8, 5))])
        return P.Agg(j, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR))])

    def numeric_join_key():
        s2 = P.SeqScan(1, [("l_quantity", P.Var(1, li.attno("l_quantity"), P.NUMERIC, 2))])
        h = P.Hash(s2, [P.out_var(s2, 1)])
        j = P.HashJoin(P.JOIN_INNER, sc, h, [P.out_var(sc, 2)], [("l_quantity", P.out_var(sc, 2))])
        return P.Agg(j, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR))])

    def bad_scanrelid():
        s9 = P.SeqScan(9, [("x", P.Var(9, 1, P.INT8))])
        return P.Agg(s9, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR))])

    ex = capi.Executor(ctx, dev)
    # HAVING compares exact aggregate states on the host: it runs (and over the no-op runtime yields no group)
    out["ran"]["having"] = {"rows": len(ex.run(having()).rows)}
    for name, build in (("sorted_agg", sorted_agg), ("sort_without_limit", sort_without_limit),
                        ("right_join", right_join), ("numeric_join_key", numeric_join_key), ("bad_scanrelid", bad_scanrelid)):
        before = ctx.launches()
        try:
            ex.run(build())
            out["refused"][name] = {"error": None}
        except capi.CbgpuError as e:
            out["refused"][name] = {"error": str(e), "code": e.code, "launches": ctx.launches() - before}
    # the executor state is reusable after a refusal
    out["ran"]["q1_after_refusals"] = {"rows": len(ex.run(tpch.q1_plan(1)).rows)}
    ex.close()

    # 3b. the round-2 host paths over the no-op runtime: outer joins through the pair probe, a sorted Gather's merge receive on a
    #     3-segment cluster, and an operator memory budget small enough for multi-batch joins and partitioned aggregation (the
    #     passes are host loops: every one of them runs, with kernels that compute nothing)
    o = rels[1]
    so = P.SeqScan(2, [("o_orderkey", P.Var(2, o.attno("o_orderkey"), P.INT8)), ("o_custkey", P.Var(2, o.attno("o_custkey"), P.INT4))])
    sl = P.SeqScan(1, [("l_orderkey", P.Var(1, li.attno("l_orderkey"), P.INT8)), ("l_suppkey", P.Var(1, li.attno("l_suppkey"), P.INT4))])
    ex = capi.Executor(ctx, dev)
    for jt, nme in ((P.JOIN_RIGHT, "right_join_runs"), (P.JOIN_FULL, "full_join_runs")):
        hh = P.Hash(so, [P.out_var(so, 1)])
        jj = P.HashJoin(jt, sl, hh, [P.out_var(sl, 1)], [("l_suppkey", P.out_var(sl, 2)), ("o_custkey", P.InnerVar(2, P.INT4))])
        before = ctx.launches()
        out["ran"][nme] = {"rows": len(ex.run(P.Agg(jj, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [("n", P.Aggref(P.AGG_COUNT_STAR))])).rows),
                           "launches": ctx.launches() - before}
    ex.close()
    exm = capi.Executor(ctx, dev, operator_mem_kb=16)
    before = ctx.launches()
    # the build side is a bare scan of orders (a base relation has its rows even here): 16 KB splits it into many batches
    hh = P.Hash(so, [P.out_var(so, 1)])
    jj = P.HashJoin(P.JOIN_INNER, sl, hh, [P.out_var(sl, 1)], [("l_suppkey", P.out_var(sl, 2)), ("o_custkey", P.InnerVar(2, P.INT4))])
    r3 = exm.run(P.Agg(jj, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("l_suppkey", P.out_var(jj, 1)), ("n", P.Aggref(P.AGG_COUNT_STAR))], num_groups=64))
    out["ran"]["q3_tiny_memory"] = {"rows": len(r3.rows), "launches": ctx.launches() - before,
                                    "batches": int(exm.estate.contents.es_hashjoin_batches_run)}
    exm.close()
    cl = capi.Cluster(ctx, [dev, dev, dev])
    before = ctx.launches()
    out["ran"]["q3_merge_gather_3seg"] = {"rows": len(cl.run(tpch.q3_plan(seg, 3, merge_gather=True)).rows), "launches": ctx.launches() - before}
    cl.close()

    # 3a. CHECK_FOR_INTERRUPTS: the callback is polled before every pipeline; pending after the 2nd poll -> the query stops with
    #     CBGPU_ERR_INTERRUPTED having launched fewer kernels than a full run, and the executor runs the next query
    import ctypes as C
    polls = {"n": 0}

    def pending(_es):
        polls["n"] += 1
        return 1 if polls["n"] > 2 else 0
    cb = C.CFUNCTYPE(C.c_int, C.c_void_p)(pending)
    ex = capi.Executor(ctx, dev)
    full = ctx.launches()
    ex.run(tpch.q5_plan(reg, 1))
    full = ctx.launches() - full
    ex.estate.contents.es_interrupt_pending = C.cast(cb, C.c_void_p)
    before = ctx.launches()
    try:
        ex.run(tpch.q5_plan(reg, 1))
        out["interrupt"] = {"code": None}
    except capi.CbgpuError as e:
        out["interrupt"] = {"code": e.code, "msg": str(e), "launches": ctx.launches() - before, "full": full, "polls": polls["n"]}
    ex.estate.contents.es_interrupt_pending = None
    out["interrupt"]["rows_after"] = len(ex.run(tpch.q5_plan(reg, 1)).rows)
    ex.close()

    # 3b. device out-of-memory at every allocation of a join query in turn: an error (never a crash), and the next run is clean
    fake = C.CDLL(None)
    fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
    ex = capi.Executor(ctx, dev)
    oom = {"failed": 0, "passed": 0, "codes": []}
    clean_in_a_row = 0
    for n in range(1, 400):
        fake.fake_cudart_fail_alloc_in(n)
        try:
            ex.run(tpch.q5_plan(reg, 1))
            oom["passed"] += 1
            clean_in_a_row += 1
        except capi.CbgpuError as e:
            oom["failed"] += 1
            clean_in_a_row = 0
            if e.code not in oom["codes"]:
                oom["codes"].append(e.code)
        fake.fake_cudart_fail_alloc_in(0)
        assert len(ex.run(tpch.q5_plan(reg, 1)).rows) == 0      # the executor state survives the failure
        if clean_in_a_row >= 3:                                  # n is past the query's last allocation
            break
    ex.close()
    out["oom"] = oom

    # 3c. the device reports an error in its status word (or hands back a word that makes no sense) at each 4-byte read-back of a
    #     join query in turn: the caller gets an error or an answer, never a crash, and the next run is clean
    fake.fake_cudart_poison_int_d2h.argtypes = [C.c_long, C.c_int]
    ex = capi.Executor(ctx, dev)
    dev_err = {"raised": 0, "returned": 0, "codes": []}
    for value in (-4, -6, -5, 0x7fffffff):
        quiet = 0
        for n in range(1, 60):
            fake.fake_cudart_poison_int_d2h(n, value)
            try:
                ex.run(tpch.q3_plan(seg, 1))
                dev_err["returned"] += 1
                quiet += 1
            except capi.CbgpuError as e:
                dev_err["raised"] += 1
                quiet = 0
                if e.code not in dev_err["codes"]:
                    dev_err["codes"].append(e.code)
            fake.fake_cudart_poison_int_d2h(0, 0)
            assert len(ex.run(tpch.q3_plan(seg, 1)).rows) == 0
            if quiet >= 4:
                break
    ex.close()
    out["device_errors"] = dev_err

    # 4. SSB Q4.x: wide group-by plans
    srels = ssb.gen_tables(0.01, capi.hashbpchar)
    if srels is not None:
        sdev = [capi.DeviceRelation.from_host(ctx, r) for r in srels]
        ex = capi.Executor(ctx, sdev)
        for q in ("q4_1", "q4_2", "q4_3"):
            out["ran"]["ssb_" + q] = {"rows": len(ex.run(getattr(ssb, q + "_plan")()).rows)}
        ex.close()
        for d in sdev:
            d.free()
    for d in dev:
        d.free()

    # 4b. the segment file loader's file handling (cb_aocs_load_segfile): reference naming, EOF bookkeeping, what is missing
    import tempfile

    import numpy as np
    from test_aocs_format import CASES
    byname = {c[0]: c for c in CASES}
    a, b = byname["int4_plain"], byname["numeric_price"]
    nrows = min(len(a[7]), len(b[7]))
    seg = {"loads": {}, "errors": {}}
    with tempfile.TemporaryDirectory() as td:
        base = os.path.join(td, "16384")
        segno = 2
        for filenum, case in ((1, a), (2, b)):
            with open(capi.aocs_segfile_path(base, segno, filenum), "wb") as f:
                f.write(case[6] + b"\0" * 100)                 # bytes past the recorded EOF exist on disk and must be ignored
        cols = [(0, 1, 4, 0, 4, 0, len(a[6])), (1, 2, -1, 1, 4, 0, len(b[6]))]
        rel = capi.DeviceRelation(ctx, max(len(a[7]), len(b[7])) + 4, [P.INT4, P.NUMERIC], dscales=[0, b[4]])

        def attempt(name, *args, **kw):
            try:
                seg["loads"][name] = list(rel.load_segfile(*args, **kw))
            except capi.CbgpuError as e:
                seg["errors"][name] = {"code": e.code, "msg": str(e)}
        if len(a[7]) == len(b[7]):
            attempt("as_recorded", base, segno, a[2], cols)
        attempt("one_column", base, segno, a[2], cols[:1])
        attempt("eof_beyond_file", base, segno, a[2], [(0, 1, 4, 0, 4, 0, len(a[6]) + 4096)])
        attempt("eof_inside_a_block", base, segno, a[2], [(0, 1, 4, 0, 4, 0, len(a[6]) - 7)])
        attempt("missing_column_file", base, segno, a[2], [(0, 5, 4, 0, 4, 0, 64)])
        attempt("missing_segno", base, 9, a[2], cols[:1])
        attempt("segno_out_of_range", base, 128, a[2], cols[:1])
        attempt("eof_zero", base, segno, a[2], [(0, 1, 4, 0, 4, 0, 0)])
        # visibility map entries are checked on the host before they go to the device: the same range twice, a first row
        # number that is not a multiple of 32 768
        empty_entry = b"\x01\0\0\0" + b"\0\0"              # version 1, no compression, zero blocks
        for name, entries in (("visimap_same_range_twice", [(0, empty_entry), (0, empty_entry)]),
                              ("visimap_misaligned_first_row", [(5, empty_entry)]),
                              ("visimap_ok", [(0, empty_entry), (32768, None)])):
            try:
                seg["loads"][name] = rel.apply_visimap(a[6], a[2], entries)
            except capi.CbgpuError as e:
                seg["errors"][name] = {"code": e.code, "msg": str(e)}
        rel.free()
    seg["rows"] = {"int4_plain": int(len(a[7])), "numeric_price": int(len(b[7]))}
    out["segfile"] = seg
    del nrows, np

    # 5. the storage side's host half: the block header walk of cbgpu_aocs_decode_column over reference-written column files,
    #    whole and damaged (bit flips, truncations), handed over in exact-size malloc'd buffers so that a sanitizer build sees any
    #    read past the file.  The kernels being no-ops, only return codes matter: no crash, no report, errors stay errors.
    if os.environ.get("CB_TEST_AOCS_FUZZ"):
        import ctypes as C

        import numpy as np
        from test_aocs_format import CASES, ZCASES, ZSTDCASES
        decode = {"int4": (P.INT4, 4, 0, 4), "int8": (P.INT8, 8, 0, 8), "date": (P.DATE, 4, 0, 4), "float8": (P.FLOAT8, 8, 0, 8),
                  "bool": (P.BOOL, 1, 0, 1), "numeric": (P.NUMERIC, -1, 1, 4), "bpchar": (P.BPCHAR1, -1, 2, 4)}
        libc = C.CDLL(None)
        libc.malloc.restype = C.c_void_p
        libc.malloc.argtypes = [C.c_size_t]
        libc.free.argtypes = [C.c_void_p]
        rng = np.random.default_rng(11)
        calls = errors = 0
        for case in CASES + ZCASES + ZSTDCASES:
            name, typname, checksum, blocksize, dscale, nblocks, raw, values, nulls = case[:9]
            kind = 0 if len(case) == 9 else (2 if name.startswith("zstd") else 1)
            ctype, attlen, varkind, align = decode[typname]
            rel = capi.DeviceRelation(ctx, len(values) + 8, [ctype], dscales=[dscale])
            variants = [raw]
            for _ in range(int(os.environ["CB_TEST_AOCS_FUZZ"])):
                bad = bytearray(raw)
                how = rng.integers(0, 3)
                if how == 0:                                    # a flipped bit in the first bytes of some 4 KB stretch: headers live there
                    pos = int(rng.integers(0, max(len(bad) // 4096, 1))) * 4096 + int(rng.integers(0, 32))
                    bad[min(pos, len(bad) - 1)] ^= 1 << int(rng.integers(0, 8))
                elif how == 1:                                  # anywhere
                    bad[int(rng.integers(0, len(bad)))] ^= 1 << int(rng.integers(0, 8))
                else:                                           # cut short
                    bad = bad[:int(rng.integers(0, len(bad)))]
                variants.append(bytes(bad))
            for v in variants:
                pin = libc.malloc(max(len(v), 1))
                C.memmove(pin, v, len(v))
                n = C.c_int64()
                rc = G.cbgpu_aocs_decode_column_ex(ctx.h, pin, len(v), 1 if checksum else 0, kind, attlen, varkind, align, rel.h, 0, 0, C.byref(n))
                libc.free(pin)
                calls += 1
                errors += 1 if rc else 0
                if v is raw:
                    assert rc == 0 and n.value == len(values), (name, rc, ctx.error())
            rel.free()
        out["aocs_fuzz"] = {"calls": calls, "errors": errors}
    ctx.close()
    # 6. partial aggregate states in the reference's serialised form (cb_numeric.c): round trips over exact-size malloc'd buffers,
    #    then the deserialiser over damaged and random bytes - under the sanitizer build any read past the buffer shows
    import ctypes as C
    import random
    E = capi.ex()
    E.cb_numeric_avg_serialize.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int32]
    E.cb_int8_avg_serialize.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int32]
    E.cb_numeric_avg_deserialize.argtypes = [C.c_void_p, C.c_int32, C.c_int32] + [C.POINTER(C.c_int64)] * 3 + [C.POINTER(C.c_int32)]
    libc = C.CDLL(None)
    libc.malloc.restype = C.c_void_p
    libc.malloc.argtypes = [C.c_size_t]
    libc.free.argtypes = [C.c_void_p]
    rnd = random.Random(5)
    ser = {"roundtrips": 0, "refused": 0, "accepted_garbage": 0}
    n_, lo_, hi_, ds_ = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    for _ in range(300):
        v = rnd.randrange(-(1 << 100), 1 << 100)
        u = v & ((1 << 128) - 1)
        lo, hi = u & ((1 << 64) - 1), u >> 64
        lo, hi = (lo - (1 << 64) if lo >= 1 << 63 else lo), (hi - (1 << 64) if hi >= 1 << 63 else hi)
        ds, cnt = rnd.randrange(0, 12), rnd.randrange(0, 1 << 40)
        tmp = C.create_string_buffer(256)
        k = E.cb_numeric_avg_serialize(cnt, lo, hi, ds, tmp, 256)
        assert k > 0
        buf = libc.malloc(k)                            # exact size: one byte too many read is a heap overflow report
        C.memmove(buf, tmp, k)
        assert E.cb_numeric_avg_deserialize(buf, k, 1, C.byref(n_), C.byref(lo_), C.byref(hi_), C.byref(ds_)) == 0
        assert (n_.value, lo_.value, hi_.value, ds_.value) == (cnt, lo, hi, ds)
        ser["roundtrips"] += 1
        for cut in (0, 1, 8, 15, 16, k - 1):            # truncations
            if cut < k and E.cb_numeric_avg_deserialize(buf, cut, 1, C.byref(n_), C.byref(lo_), C.byref(hi_), C.byref(ds_)) < 0:
                ser["refused"] += 1
        libc.free(buf)
    for _ in range(3000):
        k = rnd.randrange(0, 90)
        buf = libc.malloc(max(k, 1))
        C.memmove(buf, bytes(rnd.randrange(256) for _ in range(k)), k)
        rc = E.cb_numeric_avg_deserialize(buf, k, rnd.randrange(2), C.byref(n_), C.byref(lo_), C.byref(hi_), C.byref(ds_))
        ser["refused" if rc < 0 else "accepted_garbage"] += 1
        libc.free(buf)
    out["serialize"] = ser
    print("HOSTLOGIC " + json.dumps(out))


if __name__ == "__main__":
    main()
