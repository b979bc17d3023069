"""Worker of tests/test_host_topn_fake_runtime.py: cbgpu_topn's host loop over the no-op runtime of tests/fake_runtime.py
(LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory, so every key reads back as constant and
each call goes to the tournament).  Prints one "TOPN {json}" line per call as soon as the call returns, so that a call that never
returns is named by the lines before it.  Not a test by itself.

    host_topn_worker.py calls N      every LIMIT 1..64 over N rows, with 1 and with 4 keys
    host_topn_worker.py refusals     the calls cbgpu_topn must refuse before any launch"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402


def topn(ctx, rel, keycols, desc, uns, limit):
    n = len(keycols)
    i32 = C.c_int32 * max(n, 1)
    idx = (C.c_uint32 * 64)()
    nout = C.c_int64(-1)
    before = ctx.launches()
    rc = ctx.L.cbgpu_topn(ctx.h, rel.h, i32(*keycols), i32(*desc), i32(*uns) if uns is not None else None, n, limit, idx,
                          C.byref(nout))
    return {"rc": rc, "msg": ctx.error() if rc else "", "nout": nout.value, "launches": ctx.launches() - before}


def emit(rec):
    print("TOPN " + json.dumps(rec), flush=True)


def calls(ctx, n):
    rel = capi.DeviceRelation(ctx, n, [P.INT8] * 4, name="keys")
    for nkeys in (1, 4):
        for limit in range(1, 65):
            r = topn(ctx, rel, list(range(nkeys)), [limit & 1] * nkeys, [0] * nkeys, limit)
            emit(dict(r, n=n, nkeys=nkeys, limit=limit))
    rel.free()


def refusals(ctx):
    rel = capi.DeviceRelation(ctx, 10000, [P.INT8, P.FLOAT8, P.INT4], name="keys")
    nullable = capi.DeviceRelation(ctx, 10000, [P.INT8], name="nullable")
    zeros = bytes(8 * 10000)
    nulls = bytes(10000)
    ctx.check(ctx.L.cbgpu_rel_load_column(nullable.h, 0, zeros, nulls))
    empty = capi.DeviceRelation(ctx, 0, [P.INT8], name="empty")
    for name, r, keys, limit in (("nkeys_0", rel, [], 10), ("nkeys_5", rel, [0, 2, 0, 2, 0], 10), ("limit_0", rel, [0], 0),
                                 ("limit_65", rel, [0], 65), ("key_col_3", rel, [0, 3], 10), ("key_col_neg", rel, [-1], 10),
                                 ("float8_key", rel, [0, 1], 10), ("nullable_key", nullable, [0], 10), ("empty", empty, [0], 10),
                                 ("empty_limit_64", empty, [0, 0, 0, 0], 64)):
        emit(dict(topn(ctx, r, keys, [0] * len(keys), None, limit), name=name))
    for r in (rel, nullable, empty):
        r.free()


def main():
    ctx = capi.Context(0)
    if sys.argv[1] == "calls":
        calls(ctx, int(sys.argv[2]))
    else:
        refusals(ctx)
    ctx.close()


if __name__ == "__main__":
    main()
