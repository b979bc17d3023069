"""Worker of tests/test_host_join_filter_fake_runtime.py: the host side of the pair probe (LEFT / SEMI / ANTI hash joins with a
join filter, and INNER / FULL ones without) over tests/native/fake_cudart.c (LD_PRELOADed by the test; kernels are no-ops,
"device" memory is zeroed host memory).  Prints one JSON object.  Not a test by itself."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402
from host_batched_pairs_worker import dim, fact, scan  # noqa: E402

if os.environ.get("CB_TEST_LIBDIR"):
    capi.HERE = os.environ["CB_TEST_LIBDIR"]        # libcbgpu.so (link) + a sanitizer build of libcbexec.so

POLL = C.CFUNCTYPE(C.c_int, C.c_void_p)
JOINS = {"left": P.JOIN_LEFT, "semi": P.JOIN_SEMI, "anti": P.JOIN_ANTI, "right": P.JOIN_RIGHT, "full": P.JOIN_FULL,
         "notin": P.JOIN_LASJ_NOTIN}


def join(jointype, fo, do):
    """fact JOIN dim ON k = dk AND amt <> w"""
    sf = scan(1, fo, ["k", "amt", "g"])
    sd = scan(2, do, ["dk", "w"])
    h = P.Hash(sd, [P.out_var(sd, 1)])
    targets = [("k", P.out_var(sf, 1)), ("amt", P.out_var(sf, 2)), ("g", P.out_var(sf, 3))]
    if jointype not in (P.JOIN_SEMI, P.JOIN_ANTI, P.JOIN_LASJ_NOTIN):
        targets.append(("w", P.InnerVar(2, P.INT8)))
    return P.HashJoin(jointype, sf, h, [P.out_var(sf, 1)], targets, joinquals=[P.OpExpr(P.OP_NE, P.out_var(sf, 2), P.InnerVar(2, P.INT8))],
                      quals=[P.OpExpr(P.OP_GT, P.out_var(sf, 2), P.Const(P.INT8, 10))])


def main():
    out = {"ran": {}, "refused": {}}
    ctx = capi.Context(0)
    fo = fact(20011)
    for dup in (1, 3):
        do = dim(4000, dup)
        dev = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
        for name, t in JOINS.items():
            for mem_kb in (0, 16):
                ex = capi.Executor(ctx, dev, operator_mem_kb=mem_kb)
                before = ctx.launches()
                key = "%s_dup%d_%dkb" % (name, dup, mem_kb)
                try:
                    res = ex.run(join(t, fo, do))
                    out["ran"][key] = {"rows": len(res.rows), "launches": ctx.launches() - before,
                                       "passes": int(ex.estate.contents.es_hashjoin_batches_run),
                                       "nbatch": max(v["hashjoin_nbatch"] for v in res.instrument.values())}
                except capi.CbgpuError as e:
                    out["refused"][key] = {"code": e.code, "msg": str(e)}
                ex.close()
        for d in dev:
            d.free()

    do = dim(4000, 3)
    outer, inner = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
    L = ctx.L
    keys = (C.c_int32 * 1)(0)
    good = capi.join_filter([(outer, 1, 0), (inner, 1, 1)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_LOAD, 1, 0), (capi.CBP_NE, 0, 0)])
    ht = C.c_void_p()
    ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, 16, C.byref(ht)))
    pairs, passes = capi.CbgpuPairs(), C.c_int64()

    def probe(filt, jointype=P.JOIN_SEMI, cb=None, table=ht):
        before = ctx.launches()
        rc = L.cbgpu_ht_probe_pairs(ctx.h, table, outer.h, keys, 1, jointype, C.byref(filt) if filt is not None else None,
                                    C.cast(cb, C.c_void_p) if cb else None, None, C.byref(pairs), C.byref(passes))
        r = {"code": rc, "msg": ctx.error() if rc else "", "launches": ctx.launches() - before, "passes": passes.value,
             "npairs": pairs.npairs, "outer_idx": pairs.outer_idx}
        L.cbgpu_pairs_free(C.byref(pairs))
        return r

    out["abi_ok"] = {jt: probe(good, t) for jt, t in (("left", P.JOIN_LEFT), ("semi", P.JOIN_SEMI), ("anti", P.JOIN_ANTI))}

    # malformed descriptors and join types: refused before any launch
    bad = {
        "src2": capi.join_filter([(outer, 1, 0), (inner, 1, 2)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_LOAD, 1, 0), (capi.CBP_NE, 0, 0)]),
        "opcode_filter": capi.join_filter([(outer, 1, 0)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_FILTER, 0, 0), (capi.CBP_CONST, 0, 1)]),
        "opcode_probe": capi.join_filter([(outer, 1, 0)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_PROBE, 0, 0)]),
        "opcode_unknown": capi.join_filter([(outer, 1, 0)], [(capi.CBP_LOAD, 0, 0), (100, 0, 0)]),
        "too_deep": capi.join_filter([], [(capi.CBP_CONST, 0, 1)] * 49 + [(capi.CBP_AND, 0, 0)] * 48),
        "two_left": capi.join_filter([], [(capi.CBP_CONST, 0, 1), (capi.CBP_CONST, 0, 1)]),
        "none_left": capi.join_filter([], [(capi.CBP_CONST, 0, 1), (capi.CBP_POP, 0, 0)]),
        "underflow": capi.join_filter([], [(capi.CBP_CONST, 0, 1), (capi.CBP_NE, 0, 0)]),
        "empty": capi.join_filter([], []),
        "bad_load": capi.join_filter([(outer, 1, 0)], [(capi.CBP_LOAD, 1, 0)]),
        "bad_dup": capi.join_filter([], [(capi.CBP_DUP, 0, 0)]),
    }
    out["invalid"] = {k: probe(f) for k, f in bad.items()}
    out["invalid"]["no_filter"] = probe(None)                    # SEMI takes a filter
    for name, t in (("inner", P.JOIN_INNER), ("right", P.JOIN_RIGHT), ("full", P.JOIN_FULL), ("notin", P.JOIN_LASJ_NOTIN)):
        out["invalid"]["jointype_" + name] = probe(good, t)         # join types that take none

    # CHECK_FOR_INTERRUPTS between batches: the callback asks to stop when polled the third time
    polls = {"n": 0}

    def pending(_arg):
        polls["n"] += 1
        return 1 if polls["n"] > 2 else 0
    cb = POLL(pending)
    out["abi_interrupt"] = dict(probe(good, P.JOIN_ANTI, cb), polls=polls["n"])

    # every device allocation of the call failing in turn, with a filter and without: CBGPU_ERR_NOMEM, nothing left behind,
    # the next call clean
    fake = C.CDLL(None)
    fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
    oom = {"codes": [], "after": []}
    for jointype, filt in ((P.JOIN_SEMI, good), (P.JOIN_LEFT, good), (P.JOIN_INNER, None), (P.JOIN_FULL, None)):
        for batched in (True, False):
            table = ht
            if not batched:
                table = C.c_void_p()
                ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, 1, C.byref(table)))
            for n in range(1, 200):
                fake.fake_cudart_fail_alloc_in(n)
                r = probe(filt, jointype, table=table)
                fake.fake_cudart_fail_alloc_in(0)
                after = probe(filt, jointype, table=table)
                oom["after"].append(after["code"])
                if r["code"] == 0:
                    break
                oom["codes"].append(r["code"])
                assert r["npairs"] == 0 and r["outer_idx"] is None
            if not batched:
                L.cbgpu_ht_free(table)
    out["oom"] = oom
    L.cbgpu_ht_free(ht)
    outer.free()
    inner.free()
    ctx.close()
    print("JOINFILTER " + json.dumps(out))


if __name__ == "__main__":
    main()
