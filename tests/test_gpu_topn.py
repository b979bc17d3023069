"""The device top-N (cbgpu_topn: ORDER BY keys LIMIT n, n <= 64, csrc/agg.cu) against a plain reference: the row indices of the
first n rows when rows are sorted by their keys as Python ints, then by row index (equal keys go to the lower row, so the answer
is exact and the same on every route).  Each call's kernels are read from the launch trace to say which route ran:

    small       at most 4096 rows: k_topn_final ranks them all
    threshold   k_topn_min / k_topn_kth per leading key until one is not constant, k_topn_filter keeps the rows at or under
                the k-th smallest block minimum, k_topn_final ranks those (at most 4096)
    tournament  passes of k_topn over per-thread best-k lists: more than 4096 candidates, or every key constant

Sizes at the route boundaries, LIMITs on both sides of 32, every key type the device compares (1-byte types unsigned, int32 /
int64 limits, unsigned int8, 128-bit sums as (hi signed, lo unsigned)), every mix of ascending and descending keys, constant and
heavily tied leading keys, and the gather of the chosen rows (cbgpu_rel_take_rows).  Then Limit <- Sort over an Agg through the
executor against the oracle, including ORDER BY sum(x) DESC over groups whose sums have both signs (-m gpu)."""
import ctypes as C
import functools
import heapq

import numpy as np
import pytest

from cloudberry_b200 import capi
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from test_gpu_edge import agg_over, fact, make, run_both, scan

pytestmark = pytest.mark.gpu

I32 = (-2**31, 2**31 - 1)
I64 = (-2**63, 2**63 - 1)
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def reference(keys, desc, limit):
    """keys: one list of Python ints per sort key (already in the order the device compares them); the first `limit` row
    indices by (keys..., row index)"""
    n = len(keys[0]) if keys else 0

    def k(r):
        return tuple(-v[r] if d else v[r] for v, d in zip(keys, desc)) + (r,)
    return heapq.nsmallest(limit, range(n), key=k)


def route(names):
    """which route a cbgpu_topn call took, from its launches: (route, number of keys the threshold selection examined)"""
    if not names:
        return "none", 0
    mins = names.count("k_topn_min")
    if names == ["k_topn_final"]:
        return "small", 0
    if names == ["k_topn_min", "k_topn_kth"] * mins + ["k_topn_filter", "k_topn_final"] and mins >= 1:
        return "threshold", mins
    first = names.index("k_topn") if "k_topn" in names else len(names)
    if first < len(names) and all(x == "k_topn" for x in names[first:]):
        return "tournament", mins
    return "unknown: %s" % names, mins


def device_topn(ctx, dev, keycols, desc, uns, limit):
    n = len(keycols)
    A = C.c_int32 * n
    idx = (C.c_uint32 * 64)()
    nout = C.c_int64(-1)
    ctx.trace_begin()
    try:
        ctx.check(ctx.L.cbgpu_topn(ctx.h, dev.h, A(*keycols), A(*desc), A(*(uns or [0] * n)), n, limit, idx, C.byref(nout)))
    finally:
        names = [k for k, _ in ctx.trace_end()]
    return list(idx[:nout.value]), route(names)


def upload(ctx, types, cols):
    return capi.DeviceRelation.from_host(ctx, HostRelation("t", ["c%d" % i for i in range(len(types))], types, cols))


def check(ctx, types, cols, keycols, desc, uns, limits, ref_keys=None):
    """device answer == reference for every limit; returns the routes taken"""
    dev = upload(ctx, types, cols)
    if ref_keys is None:
        ref_keys = []
        for c, u in zip(keycols, uns or [0] * len(keycols)):
            vals = cols[c].tolist()
            ref_keys.append([v & M64 for v in vals] if u else vals)
        ref_desc = desc
    else:
        ref_keys, ref_desc = ref_keys
    want = reference(ref_keys, ref_desc, max(limits))
    routes = []
    try:
        for limit in limits:
            got, r = device_topn(ctx, dev, keycols, desc, uns, limit)
            assert got == want[:limit], (limit, r, got[:8], want[:8])
            routes.append(r)
    finally:
        dev.free()
    return routes


# --- sizes x limits ----------------------------------------------------------------------------------------------------------
LIMITS = [1, 2, 31, 32, 33, 63, 64]


@functools.lru_cache(maxsize=None)
def _sized(n):
    """(columns, the first 64 rows): a shorter LIMIT's answer is a prefix of it, the order being total"""
    rng = np.random.default_rng(1000 + n)
    cols = [rng.integers(-50000, 50001, n).astype(np.int32), rng.integers(I64[0], I64[1], n, endpoint=True)]
    return cols, reference([c.tolist() for c in cols], [0, 1], 64)


@pytest.mark.parametrize("limit", LIMITS)
@pytest.mark.parametrize("size", [0, 1, "limit-1", "limit", "limit+1", 4096, 4097, 16128, 16129, 10**5, 10**6])
def test_sizes_and_limits(ctx, size, limit):
    """an INT4 key with ties, then an INT8 key descending: at most 4096 rows are ranked at once, above that the threshold
    selection decides - at 4097 to 16 128 rows too, where LIMIT 64 has fewer blocks of 256 rows than it needs"""
    n = {"limit-1": limit - 1, "limit": limit, "limit+1": limit + 1}.get(size, size)
    cols, want = _sized(n)
    dev = upload(ctx, [P.INT4, P.INT8], cols)
    try:
        got, r = device_topn(ctx, dev, [0, 1], [0, 1], None, limit)
    finally:
        dev.free()
    assert got == want[:limit], (n, r, got[:8], want[:8])
    assert r == (("none", 0) if n == 0 else ("small", 0) if n <= 4096 else ("threshold", 1)), (n, r)


# --- key types ---------------------------------------------------------------------------------------------------------------
def _typed(typ, n, rng):
    if typ in (P.INT4, P.DATE):
        lo, hi = I32
        special = [lo, lo + 1, -1, 0, 1, hi - 1, hi]
        v = rng.integers(lo, hi, n, endpoint=True)
    elif typ in (P.INT8, P.NUMERIC):
        lo, hi = I64
        special = [lo, lo + 1, -1, 0, 1, hi - 1, hi]
        v = rng.integers(lo, hi, n, endpoint=True)
    elif typ == P.DICT32:
        special = [0, 1, 2**31 - 2, 2**31 - 1]
        v = np.where(rng.random(n) < 0.5, rng.integers(0, 1000, n), rng.integers(0, 2**31, n))
    else:                                   # DICT8, BPCHAR1, BOOL: bytes, compared unsigned
        special = [0, 127, 128, 255]
        v = rng.integers(0, 256, n)
    v = v.astype(np.int64)
    for s in special:                        # three copies of each: ties at the extremes go to the lower row
        v[rng.choice(n, 3, replace=False)] = s
    return v


@pytest.mark.parametrize("n", [3000, 50000])
@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("typ", [P.INT4, P.DATE, P.INT8, P.NUMERIC, P.DICT32, P.DICT8, P.BPCHAR1, P.BOOL])
def test_key_types(ctx, typ, desc, n):
    rng = np.random.default_rng(typ * 10 + desc + n)
    v = _typed(typ, n, rng)
    routes = check(ctx, [typ], [v], [0], [desc], None, [1, 33, 64])
    for r in routes:
        assert r == ("small", 0) if n <= 4096 else r[0] in ("threshold", "tournament"), routes


# --- key shapes --------------------------------------------------------------------------------------------------------------
MIXES = [tuple((m >> i) & 1 for i in range(k)) for k in range(1, 5) for m in range(1 << k)]


@pytest.mark.parametrize("n", [20000, 100000])
@pytest.mark.parametrize("desc", MIXES, ids=lambda d: "".join("d" if x else "a" for x in d))
def test_ascending_descending_mixes(ctx, desc, n):
    """1 to 4 keys, each ascending or descending: a leading INT4 of 7 values (about n / 7 rows tie on it: under 4096 at 20 000
    rows, over 4096 at 100 000), then a few-valued INT8, a DICT8 and a NUMERIC of both signs"""
    rng = np.random.default_rng(sum(d << i for i, d in enumerate(desc)) * 7 + len(desc) * 1000 + n)
    cols = [rng.integers(-3, 4, n), rng.integers(-5, 5, n), rng.integers(0, 256, n), rng.integers(-10**12, 10**12, n)]
    types = [P.INT4, P.INT8, P.DICT8, P.NUMERIC]
    k = len(desc)
    routes = check(ctx, types, cols, list(range(k)), list(desc), None, [33, 64])
    want = ("threshold", 1) if n == 20000 else "tournament"
    assert all((r if n == 20000 else r[0]) == want for r in routes), routes


@pytest.mark.parametrize("n", [3000, 20000, 50000])
@pytest.mark.parametrize("desc", [0, 1])
def test_unsigned_int8_with_the_top_bit_set(ctx, desc, n):
    """unsigned_cmp on an INT8 holding 0, 1, 2^63 - 1, 2^63, 2^63 + 1 and 2^64 - 1 (stored as negative int64s), then an INT4:
    ranked, selected by threshold and by tournament (n / 6 ties on the leading key)"""
    rng = np.random.default_rng(300 + desc + n)
    k0 = rng.choice(np.array([0, 1, 2**63 - 1, -2**63, -2**63 + 1, -1], dtype=np.int64), n)
    k1 = rng.integers(I32[0], I32[1], n)
    routes = check(ctx, [P.INT8, P.INT4], [k0, k1], [0, 1], [desc, 1 - desc], [1, 0], [1, 32, 33, 64])
    want = {3000: "small", 20000: "threshold", 50000: "tournament"}[n]
    assert all(r[0] == want for r in routes), routes


@pytest.mark.parametrize("desc", [0, 1])
def test_unsigned_int8_full_range(ctx, desc):
    rng = np.random.default_rng(310 + desc)
    k0 = rng.integers(I64[0], I64[1], 10**6, endpoint=True)
    routes = check(ctx, [P.INT8], [k0], [0], [desc], [1], [1, 64])
    assert all(r == ("threshold", 1) for r in routes), routes


# --- 128-bit sums as (hi signed, lo unsigned) --------------------------------------------------------------------------------
def _pairs(vals):
    hi = np.array([v >> 64 for v in vals], dtype=np.int64)
    lo = np.array([(v & M64) - (1 << 64) if v & (1 << 63) else v & M64 for v in vals], dtype=np.int64)
    return hi, lo


@pytest.mark.parametrize("n", [3000, 50000, 10**6])
@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("hi_kind", ["varies", "zero", "minus_one"])
def test_128_bit_pairs(ctx, hi_kind, desc, n):
    """values around 0, +-2^63 and +-2^64 split into (hi, lo) and ordered against the Python int hi * 2^64 + lo.  With a constant
    hi (every value in [0, 2^64) or in [-2^64, 0)) the threshold selection skips it and selects on lo"""
    rng = np.random.default_rng({"varies": 0, "zero": 1, "minus_one": 2}[hi_kind] * 100 + desc * 10 + n % 97)
    if hi_kind == "varies":
        centers = [0, 2**63, -2**63, 2**64, -2**64]
        base = [centers[i] for i in rng.integers(0, len(centers), n).tolist()]
        vals = [b + o for b, o in zip(base, rng.integers(-3000, 3000, n).tolist())]
    else:
        vals = [int(x) for x in rng.integers(0, 2**64, n, dtype=np.uint64)]
        for i, s in zip(rng.choice(n, 8, replace=False).tolist(), [0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1, 5]):
            vals[i] = s
        if hi_kind == "minus_one":
            vals = [v - 2**64 for v in vals]
    hi, lo = _pairs(vals)
    assert [int(h) * 2**64 + (int(lv) & M64) for h, lv in zip(hi[:50], lo[:50])] == vals[:50]
    routes = check(ctx, [P.INT8, P.INT8], [hi, lo], [0, 1], [desc, desc], [0, 1], [1, 33, 64], ref_keys=([vals], [desc]))
    for r in routes:
        if n <= 4096:
            assert r == ("small", 0), routes
        elif hi_kind != "varies":
            assert r == ("threshold", 2), routes          # hi is constant: skipped, lo decides
        else:
            assert r[0] in ("threshold", "tournament"), routes


# --- constant and heavily tied leading keys ----------------------------------------------------------------------------------
@pytest.mark.parametrize("nconst", [1, 2, 3])
@pytest.mark.parametrize("desc", [0, 1])
def test_constant_leading_keys(ctx, nconst, desc):
    """1 to 3 constant keys (INT4, DICT8 above 127, negative NUMERIC) before a varying INT8: each is examined and skipped"""
    n = 50000
    rng = np.random.default_rng(400 + nconst * 2 + desc)
    consts = [np.full(n, 7), np.full(n, 200), np.full(n, -5)][:nconst]
    cols = consts + [rng.integers(I64[0], I64[1], n, endpoint=True)]
    types = [P.INT4, P.DICT8, P.NUMERIC][:nconst] + [P.INT8]
    routes = check(ctx, types, cols, list(range(nconst + 1)), [desc] * (nconst + 1), None, [1, 33, 64])
    assert all(r == ("threshold", nconst + 1) for r in routes), routes


@pytest.mark.parametrize("n", [4097, 50000])
def test_all_keys_constant(ctx, n):
    """nothing decides but the row index: the tournament returns rows 0 .. limit - 1"""
    cols = [np.full(n, -3), np.full(n, 9)]
    routes = check(ctx, [P.INT8, P.BOOL], cols, [0, 1], [1, 0], None, [1, 32, 33, 64])
    assert all(r == ("tournament", 2) for r in routes), routes
    dev = upload(ctx, [P.INT8, P.BOOL], cols)
    got, _ = device_topn(ctx, dev, [0, 1], [0, 0], None, 64)
    dev.free()
    assert got == list(range(64))


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("ntied", [4095, 4096, 4097, 5000])
def test_tied_leading_key_at_the_candidate_limit(ctx, ntied, desc):
    """ntied rows share the leading key's first value and a second key orders them: up to 4096 candidates are ranked after the
    threshold selection, 4097 and more go to the tournament"""
    n = 100000
    rng = np.random.default_rng(500 + ntied + desc)
    k0 = rng.integers(0, 10**6, n)
    k0[rng.choice(n, ntied, replace=False)] = 10**7 if desc else -7
    k1 = rng.integers(I64[0], I64[1], n, endpoint=True)
    routes = check(ctx, [P.INT4, P.INT8], [k0, k1], [0, 1], [desc, 0], None, [1, 33, 64])
    want = ("threshold", 1) if ntied <= 4096 else ("tournament", 1)
    assert all(r == want for r in routes), routes


# --- the gather of the chosen rows -------------------------------------------------------------------------------------------
def test_take_rows_over_every_column_type(ctx):
    """cbgpu_rel_take_rows with the indices the top-N chose: every column type (the 16-byte numeric128 too) and NULL maps, against
    a numpy take"""
    L = ctx.L
    n = 50000
    rng = np.random.default_rng(600)
    spec = [(P.INT8, np.int64, rng.integers(I64[0], I64[1], n, endpoint=True)), (P.INT4, np.int32, rng.integers(I32[0], I32[1], n)),
            (P.DATE, np.int32, rng.integers(-5000, 5000, n)), (P.NUMERIC, np.int64, rng.integers(-10**15, 10**15, n)),
            (P.BPCHAR1, np.uint8, rng.integers(0, 256, n)), (P.DICT8, np.uint8, rng.integers(0, 256, n)),
            (P.DICT32, np.int32, rng.integers(0, 2**31, n)), (P.FLOAT8, np.float64, rng.normal(0, 1e6, n)),
            (P.BOOL, np.uint8, rng.integers(0, 2, n)), (P.NUMERIC128, np.int64, rng.integers(I64[0], I64[1], (n, 2), endpoint=True))]
    types = [t for t, _, _ in spec]
    cols = [np.ascontiguousarray(v, dtype=dt) for _, dt, v in spec]
    nulls = [None] + [(rng.random(n) < 0.2).astype(np.uint8) if i % 2 else None for i in range(1, len(spec))]
    src = capi.DeviceRelation(ctx, n, types, name="src")
    for i, (c, nl) in enumerate(zip(cols, nulls)):
        ctx.check(L.cbgpu_rel_load_column(src.h, i, c.ctypes.data, nl.ctypes.data if nl is not None else None))
    for limit in (1, 64):
        got, r = device_topn(ctx, src, [0], [1], None, limit)
        assert got == reference([cols[0].tolist()], [1], limit) and r == ("threshold", 1)
        idx = np.array(got, dtype=np.uint32)
        didx = C.c_void_p()
        ctx.check(L.cbgpu_dev_alloc(ctx.h, idx.nbytes, C.byref(didx)))
        ctx.check(L.cbgpu_dev_write(ctx.h, didx, idx.nbytes, idx.ctypes.data))
        dst = capi.DeviceRelation(ctx, limit, types, name="dst")
        ctx.check(L.cbgpu_rel_take_rows(dst.h, src.h, didx, limit))
        for i, (c, nl) in enumerate(zip(cols, nulls)):
            out = np.zeros((limit,) + c.shape[1:], dtype=c.dtype)
            onull = np.full(limit, 7, dtype=np.uint8)
            ctx.check(L.cbgpu_rel_read_column(dst.h, i, 0, limit, out.ctypes.data, onull.ctypes.data))
            assert np.array_equal(out.view(np.uint8), c[idx].view(np.uint8)), (i, types[i])
            assert np.array_equal(onull, nl[idx] if nl is not None else np.zeros(limit, dtype=np.uint8)), (i, types[i])
        dst.free()
        L.cbgpu_dev_free(ctx.h, didx)
    src.free()


# --- Limit <- Sort over an Agg through the executor --------------------------------------------------------------------------
ORDERS = {
    # (agg group keys, aggregates, sort keys over the Agg's targets [(attno, descending)])
    "sum_v_desc": (["k"], [("s", P.AGG_SUM, "v"), ("n", P.AGG_COUNT_STAR, None)], [(2, True), (1, False)]),
    "count_desc": (["k"], [("s", P.AGG_SUM, "v"), ("n", P.AGG_COUNT_STAR, None)], [(3, True), (1, False)]),
    "g_count_desc": (["g", "k"], [("n", P.AGG_COUNT_STAR, None)], [(1, False), (3, True), (2, False)]),
    "sum_amt": (["k"], [("s", P.AGG_SUM, "amt")], [(2, False), (1, False)]),
}


def _expected_route(order, groups):
    """the route the data forces, where it does: None where either selection route may run"""
    if groups <= 4096:
        return "small"
    if order == "sum_amt":
        return "threshold"                   # amt >= 0: the sums' hi is constant, lo is (almost) distinct
    if order == "sum_v_desc":
        return "threshold" if groups < 6000 else "tournament"      # about half the groups sum to >= 0: hi = 0 ties on them
    if order == "g_count_desc":
        return "threshold" if -(-groups // 7) <= 4096 else "tournament"    # the groups with g = 0 tie on the leading key
    return None


@pytest.mark.parametrize("order", list(ORDERS))
@pytest.mark.parametrize("groups", [4096, 4097, 16128, 16129, 50000])
def test_limit_sort_over_agg_through_the_executor(ctx, oracle, groups, order):
    """exactly `groups` groups (k = 0 .. groups - 1, g = k % 7 a DICT8), v an INT8 of both signs, amt a numeric >= 0; every sort
    ends with the unique k, so the order is total and the oracle's rows match in order"""
    n = groups * 6
    fo, fp = make(fact, n, seed=groups)
    k = np.random.default_rng(groups).permutation(np.arange(n) % groups)
    for rel in (fo, fp):
        rel.columns[0][:] = k
        rel.columns[4][:] = k % 7
    names = ["k", "v", "amt", "g"]
    gkeys, aggs, sort_keys = ORDERS[order]
    agg = agg_over(scan(1, fo, names), names, gkeys, aggs)
    agg.numGroups = groups                   # the planner's estimate: the hash table is sized once
    want_route = _expected_route(order, groups)
    for limit in (1, 10, 33, 64):
        ctx.trace_begin()
        try:
            got, want = run_both(ctx, oracle, P.LimitSort(agg, sort_keys, limit), [fo], [fp], False)
        finally:
            trace = [x for x, _ in ctx.trace_end() if x.startswith("k_topn")]
        assert len(want) == limit
        assert [tuple(map(str, r)) for r in got] == [tuple(map(str, r)) for r in want], (limit, got[:3], want[:3])
        r = route(trace)[0]
        assert r == want_route if want_route else r in ("threshold", "tournament"), (limit, trace)
