"""Worker of tests/test_host_batched_pairs_fake_runtime.py: the host side of pair joins over a build side split into batches,
driven over the no-op runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed
host memory).  Prints one JSON object.  Not a test by itself."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402
from cloudberry_b200.relation import HostRelation  # noqa: E402

POLL = C.CFUNCTYPE(C.c_int, C.c_void_p)


def fact(n):
    import numpy as np
    rng = np.random.default_rng(1)
    return HostRelation("fact", ["k", "amt", "g"], [P.INT4, P.INT8, P.INT4],
                        [rng.integers(0, 3000, n).astype(np.int32), rng.integers(0, 1000, n), rng.integers(0, 7, n).astype(np.int32)],
                        nulls=[(rng.random(n) < 0.1).astype(np.uint8), None, None])


def dim(n, dup):
    import numpy as np
    rng = np.random.default_rng(2)
    keys = np.repeat(rng.permutation(3000)[:n // dup], dup)[:n].astype(np.int32)
    return HostRelation("dim", ["dk", "w"], [P.INT4, P.INT8], [keys, rng.integers(0, 100, len(keys))],
                        nulls=[(rng.random(len(keys)) < 0.1).astype(np.uint8), None])


def scan(relid, rel, names):
    return P.SeqScan(relid, [(nme, P.Var(relid, *rel.var(nme))) for nme in names])


def join(jointype, fo, do):
    sf = scan(1, fo, ["k", "amt", "g"])
    sd = scan(2, do, ["dk", "w"])
    h = P.Hash(sd, [P.out_var(sd, 1)])
    return P.HashJoin(jointype, sf, h, [P.out_var(sf, 1)],
                      [("k", P.out_var(sf, 1)), ("amt", P.out_var(sf, 2)), ("g", P.out_var(sf, 3)), ("w", P.InnerVar(2, P.INT8))])


def agg(j):
    v = lambda i: P.out_var(j, i)  # noqa: E731
    return P.Agg(j, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [3], [("g", v(3)), ("n", P.Aggref(P.AGG_COUNT_STAR)), ("sw", P.Aggref(P.AGG_SUM, v(4)))],
                 num_groups=16)


def main():
    out = {"ran": {}}
    ctx = capi.Context(0)
    fo = fact(20011)
    jt = {"inner": P.JOIN_INNER, "left": P.JOIN_LEFT, "right": P.JOIN_RIGHT, "full": P.JOIN_FULL}
    for dup in (1, 3):
        do = dim(4000, dup)
        dev = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
        for name, t in jt.items():
            for shape, plan in (("rows", join(t, fo, do)), ("agg", agg(join(t, fo, do)))):
                ex = capi.Executor(ctx, dev, operator_mem_kb=16)
                before = ctx.launches()
                res = ex.run(plan)
                out["ran"]["%s_dup%d_%s" % (name, dup, shape)] = {
                    "rows": len(res.rows), "launches": ctx.launches() - before,
                    "passes": int(ex.estate.contents.es_hashjoin_batches_run),
                    "nbatch": max(v["hashjoin_nbatch"] for v in res.instrument.values())}
                ex.close()
        for d in dev:
            d.free()

    # CHECK_FOR_INTERRUPTS between the batches of a pair join, through the C ABI: the callback asks to stop when polled the
    # third time, i.e. after the second batch
    do = dim(4000, 3)
    outer, inner = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
    L = ctx.L
    keys = (C.c_int32 * 1)(0)
    ht = C.c_void_p()
    ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, 16, C.byref(ht)))
    pairs = capi.CbgpuPairs()
    passes = C.c_int64()
    before = ctx.launches()
    ctx.check(L.cbgpu_ht_probe_pairs(ctx.h, ht, outer.h, keys, 1, P.JOIN_FULL, None, None, None, C.byref(pairs), C.byref(passes)))
    full = {"launches": ctx.launches() - before, "passes": passes.value}
    L.cbgpu_pairs_free(C.byref(pairs))
    polls = {"n": 0}

    def pending(_arg):
        polls["n"] += 1
        return 1 if polls["n"] > 2 else 0
    cb = POLL(pending)
    before = ctx.launches()
    rc = L.cbgpu_ht_probe_pairs(ctx.h, ht, outer.h, keys, 1, P.JOIN_FULL, None, C.cast(cb, C.c_void_p), None, C.byref(pairs),
                                C.byref(passes))
    out["abi_interrupt"] = {"code": rc, "msg": ctx.error(), "launches": ctx.launches() - before, "passes": passes.value,
                            "polls": polls["n"], "npairs": pairs.npairs, "outer_idx": pairs.outer_idx, "full": full}
    ctx.check(L.cbgpu_ht_probe_pairs(ctx.h, ht, outer.h, keys, 1, P.JOIN_RIGHT, None, None, None, C.byref(pairs), C.byref(passes)))
    out["abi_after"] = {"passes": passes.value}
    L.cbgpu_pairs_free(C.byref(pairs))
    L.cbgpu_ht_free(ht)
    outer.free()
    inner.free()

    # the executor polls es_interrupt_pending once per batch of the pair join (on top of its per-pipeline polls); stopping at
    # any one of them ends the query with CBGPU_ERR_INTERRUPTED, and the executor runs the next query
    dev = [capi.DeviceRelation.from_host(ctx, r) for r in (fo, do)]
    plan = agg(join(P.JOIN_FULL, fo, do))

    def count_polls(mem_kb):
        n = {"n": 0}
        f = POLL(lambda _es: n.__setitem__("n", n["n"] + 1) or 0)
        ex = capi.Executor(ctx, dev, operator_mem_kb=mem_kb)
        ex.estate.contents.es_interrupt_pending = C.cast(f, C.c_void_p)
        before = ctx.launches()
        res = ex.run(plan)
        nb = max(v["hashjoin_nbatch"] for v in res.instrument.values())
        ex.close()
        return n["n"], ctx.launches() - before, nb
    p0, _, _ = count_polls(0)
    p1, full_launches, nbatch = count_polls(16)
    sweep = {"codes": [], "launches": [], "rows_after": []}
    for k in range(1, p1 + 1):
        n = {"n": 0}
        f = POLL(lambda _es, k=k: 1 if n.__setitem__("n", n["n"] + 1) or n["n"] >= k else 0)
        ex = capi.Executor(ctx, dev, operator_mem_kb=16)
        ex.estate.contents.es_interrupt_pending = C.cast(f, C.c_void_p)
        before = ctx.launches()
        try:
            ex.run(plan)
            sweep["codes"].append(0)
        except capi.CbgpuError as e:
            sweep["codes"].append(e.code)
        sweep["launches"].append(ctx.launches() - before)
        ex.estate.contents.es_interrupt_pending = None
        sweep["rows_after"].append(len(ex.run(plan).rows))
        ex.close()
    out["exec_interrupt"] = {"polls_unsplit": p0, "polls_split": p1, "nbatch": nbatch, "full_launches": full_launches, **sweep}
    for d in dev:
        d.free()
    ctx.close()
    print("BATCHEDPAIRS " + json.dumps(out))


if __name__ == "__main__":
    main()
