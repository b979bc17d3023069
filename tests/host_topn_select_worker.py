"""Worker of tests/test_host_topn_select_fake_runtime.py: cbgpu_topn_select's host side over the no-op runtime of
tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory, so the image pass
reads back no varying digit and each call takes its rows through k_tsel_finish).  Prints one "TSEL {json}" line per call.
Not a test by itself.

    host_topn_select_worker.py calls N      LIMITs 1, 64, 65, 100, 4096 and 10^6 over N rows, with 1 and with 4 keys
    host_topn_select_worker.py refusals     the calls cbgpu_topn_select must refuse before any launch
    host_topn_select_worker.py frees N      every device allocation of one call over N rows fails in turn"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402

LIMITS = (1, 64, 65, 100, 4096, 10**6)


def select(ctx, rel, keys, limit):
    arr = (capi.CbgpuSortKey * max(len(keys), 1))(*[capi.CbgpuSortKey(**k) for k in keys])
    idx = (C.c_uint32 * max(1, min(max(limit, 0), rel.nrows)))()
    nout = C.c_int64(-1)
    before = ctx.launches()
    rc = ctx.L.cbgpu_topn_select(ctx.h, rel.h, arr, len(keys), limit, idx, C.byref(nout))
    return {"rc": rc, "msg": ctx.error() if rc else "", "nout": nout.value, "launches": ctx.launches() - before}


def emit(rec):
    print("TSEL " + json.dumps(rec), flush=True)


def four_keys(nkeys):
    """an int8 key over the NULL map of column 0, a float8 key, an unsigned key and one whose NULLs are an N column"""
    keys = [dict(col=0, nulls=capi.SORT_NULLS_MAP), dict(col=1, float8=1, descending=1), dict(col=2, unsigned_cmp=1),
            dict(col=2, nulls=capi.SORT_NULLS_COUNT, null_col=3, descending=1)]
    return keys[:nkeys]


def keys_rel(ctx, n):
    rel = capi.DeviceRelation(ctx, n, [P.INT8, P.FLOAT8, P.INT8, P.INT8], name="keys")
    ctx.check(ctx.L.cbgpu_rel_load_column(rel.h, 0, bytes(8 * n), bytes(n)))
    return rel


def calls(ctx, n):
    rel = keys_rel(ctx, n)
    for nkeys in (1, 4):
        for limit in LIMITS:
            emit(dict(select(ctx, rel, four_keys(nkeys), limit), n=n, nkeys=nkeys, limit=limit))
    rel.free()


def refusals(ctx):
    rel = capi.DeviceRelation(ctx, 10000, [P.INT8, P.FLOAT8, P.INT4, P.NUMERIC128], name="keys")
    empty = capi.DeviceRelation(ctx, 0, [P.INT8], name="empty")
    count = capi.SORT_NULLS_COUNT
    for name, r, keys, limit in (
            ("nkeys_0", rel, [], 10), ("nkeys_5", rel, [dict(col=0)] * 5, 10), ("limit_0", rel, [dict(col=0)], 0),
            ("limit_neg", rel, [dict(col=0)], -1), ("key_col_4", rel, [dict(col=0), dict(col=4)], 10),
            ("key_col_neg", rel, [dict(col=-1)], 10), ("key_128bit", rel, [dict(col=3)], 10),
            ("float8_on_int4", rel, [dict(col=2, float8=1)], 10),
            ("null_col_float8", rel, [dict(col=0, nulls=count, null_col=1)], 10),
            ("null_col_int4", rel, [dict(col=0, nulls=count, null_col=2)], 10),
            ("null_col_out", rel, [dict(col=0, nulls=count, null_col=7)], 10),
            ("null_source_bad", rel, [dict(col=0, nulls=9)], 10),
            ("empty", empty, [dict(col=0)], 10), ("empty_limit_10e6", empty, [dict(col=0)] * 4, 10**6)):
        emit(dict(select(ctx, r, keys, limit), name=name))
    for r in (rel, empty):
        r.free()


def frees(ctx, n):
    """fail the k-th device allocation of one call, k = 1, 2, ... until the call succeeds: each failure is CBGPU_ERR_NOMEM and
    leaves no allocation behind"""
    fake = C.CDLL(None)
    fake.fake_cudart_fail_alloc_in.argtypes = [C.c_long]
    fake.fake_cudart_live_allocs.restype = C.c_long
    rel = keys_rel(ctx, n)
    for limit in (100, n):
        k, codes, leaks = 0, [], []
        while True:
            k += 1
            base = fake.fake_cudart_live_allocs()
            fake.fake_cudart_fail_alloc_in(k)
            r = select(ctx, rel, four_keys(4), limit)
            fake.fake_cudart_fail_alloc_in(0)
            if fake.fake_cudart_live_allocs() != base:
                leaks.append([k, fake.fake_cudart_live_allocs() - base])
            if r["rc"] == 0:
                break
            codes.append(r["rc"])
        emit(dict(name="frees_limit_%d" % limit, failed=k - 1, codes=sorted(set(codes)), leaks=leaks, nout=r["nout"]))
    rel.free()


def main():
    ctx = capi.Context(0)
    if sys.argv[1] == "calls":
        calls(ctx, int(sys.argv[2]))
    elif sys.argv[1] == "frees":
        frees(ctx, int(sys.argv[2]))
    else:
        refusals(ctx)
    ctx.close()


if __name__ == "__main__":
    main()
