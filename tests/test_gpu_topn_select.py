"""The device top-N for any LIMIT (cbgpu_topn_select, csrc/agg.cu) against a numpy reference that sorts stably by the keys,
so equal keys keep row order: NULLs last ascending and first descending, float8 as float8_cmp_internal orders it (every NaN
equal and above +Infinity, -0 = +0), unsigned keys as unsigned.  LIMITs around 64 and 4096, up to 65 537 and the row count
itself, over 0 to 10^7 rows; every key type and direction, 128-bit (hi, lo) pairs, NULL maps dense, sparse, all-NULL and none,
N-column NULL sources, float8 specials, constant and heavily tied keys.  The launch trace shows the route: the image pass, three
kernels per varying digit to select (none when the LIMIT takes every row), k_tsel_finish, three per varying digit to sort.
Then Limit <- Sort through the executor against the oracle over keys cbgpu_topn does not take, and TPC-H Q21 at its own LIMIT
100 (-m gpu)."""
import functools

import numpy as np
import pytest

from cloudberry_b200 import capi, tpch_q21
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import to_device
from test_gpu_edge import agg_over, dim, fact, make, run_both, scan

pytestmark = pytest.mark.gpu

NONE, MAP, COUNT = capi.SORT_NULLS_NONE, capi.SORT_NULLS_MAP, capi.SORT_NULLS_COUNT


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _order_arrays(col, null, key):
    """numpy arrays whose ascending lexicographic order is this key's order (most significant first)"""
    n = len(col)
    desc = key.get("descending", 0)
    isnull = np.zeros(n, dtype=bool) if null is None else null.astype(bool)
    if key.get("float8"):
        f = col.view(np.float64) if col.dtype != np.float64 else col
        nan = np.isnan(f) & ~isnull
        v = np.where(nan | isnull, 0.0, f) + 0.0          # -0 + 0.0 = +0
        parts = [nan.astype(np.int8), v]
        if desc:
            parts = [-parts[0], -parts[1]]
    else:
        v = col.astype(np.int64)
        if key.get("unsigned_cmp"):
            v = v.view(np.uint64)
        v = np.where(isnull, np.zeros(1, dtype=v.dtype), v)
        parts = [~v if desc else v]
    flag = (isnull != bool(desc)).astype(np.int8)
    return [flag] + parts


def reference(cols, nulls, keys, limit):
    arrays = []
    for k in keys:
        if k.get("nulls") == MAP:
            null = nulls[k["col"]]
        elif k.get("nulls") == COUNT:
            null = cols[k["null_col"]] == 0
        else:
            null = None
        arrays += _order_arrays(cols[k["col"]], null, k)
    if not len(cols[0]):
        return []
    order = np.lexsort(arrays[::-1]) if arrays else np.arange(len(cols[0]))
    return order[:limit].tolist()


def upload(ctx, types, cols, nulls=None):
    return capi.DeviceRelation.from_host(ctx, HostRelation("t", ["c%d" % i for i in range(len(types))], types, cols, nulls=nulls))


def device(ctx, dev, keys, limit):
    ctx.trace_begin()
    try:
        got = capi.topn_select(ctx, dev, keys, limit)
    finally:
        names = [k for k, _ in ctx.trace_end()]
    return got, names


def route_ok(names, n, limit):
    """image, select passes (none when every row is taken), finish, sort passes: one count / plan / scatter per varying digit"""
    if n == 0:
        return names == []
    assert names[0] == "k_tsel_image" and "k_tsel_finish" in names, names
    f = names.index("k_tsel_finish")
    sel, srt = names[1:f], names[f + 1:]
    triple = ["k_tsel_count", "k_tsel_plan", "k_tsel_scatter"]
    assert len(srt) % 3 == 0 and srt == triple * (len(srt) // 3), names
    assert sel == (triple * (len(srt) // 3) if limit < n else []), names
    return True


def check(ctx, types, cols, keys, limits, nulls=None):
    dev = upload(ctx, types, cols, nulls)
    n = len(cols[0])
    want = reference(cols, nulls or [None] * len(cols), keys, max(limits))
    try:
        for limit in limits:
            got, names = device(ctx, dev, keys, limit)
            assert got == want[:limit], (n, limit, got[:8], want[:8])
            assert route_ok(names, n, limit)
    finally:
        dev.free()


# --- sizes x limits ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _sized(n):
    rng = np.random.default_rng(7000 + n)
    return [rng.integers(-5000, 5001, n).astype(np.int32), rng.integers(-2**63, 2**63 - 1, n, endpoint=True)]


@pytest.mark.parametrize("n", [0, 1, 64, 65, 100, 4097, 65537, 10**6, 10**7])
def test_sizes_and_limits(ctx, n):
    """an INT4 key with ties, then an INT8 key descending"""
    limits = sorted({1, 64, 65, 100, 4096, 65537, max(n - 1, 1), max(n, 1), n + 1})
    check(ctx, [P.INT4, P.INT8], _sized(n), [dict(col=0), dict(col=1, descending=1)], limits)


# --- key types and directions ------------------------------------------------------------------------------------------------
def _typed(typ, n, rng):
    if typ in (P.INT4, P.DATE):
        v = rng.integers(-2**31, 2**31 - 1, n, endpoint=True)
        v[:7] = [-2**31, -2**31 + 1, -1, 0, 1, 2**31 - 2, 2**31 - 1]
        return v.astype(np.int32)
    if typ in (P.INT8, P.NUMERIC):
        v = rng.integers(-2**63, 2**63 - 1, n, endpoint=True)
        v[:5] = [-2**63, -1, 0, 1, 2**63 - 1]
        return v
    return rng.integers(0, 256, n).astype(np.uint8)


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("typ", [P.INT4, P.DATE, P.INT8, P.NUMERIC, P.BPCHAR1, "uint64"])
def test_key_types(ctx, typ, desc):
    n = 200003
    rng = np.random.default_rng(typ if isinstance(typ, int) else 99)
    if typ == "uint64":
        col, key = _typed(P.INT8, n, rng), dict(col=0, unsigned_cmp=1, descending=desc)
        typ = P.INT8
    else:
        col, key = _typed(typ, n, rng), dict(col=0, descending=desc)
    check(ctx, [typ], [col], [key], [1, 65, 4096, n])


@pytest.mark.parametrize("desc", [(0, 0), (1, 1), (0, 1)])
def test_128_bit_pairs(ctx, desc):
    """(hi signed, lo unsigned) as the executor orders exact sums: hi mostly 0 / -1, lo anywhere"""
    n = 300000
    rng = np.random.default_rng(11)
    hi = rng.choice(np.array([-1, 0, 0, 1, -2**63, 2**63 - 1]), n)
    lo = rng.integers(-2**63, 2**63 - 1, n, endpoint=True)
    keys = [dict(col=0, descending=desc[0]), dict(col=1, unsigned_cmp=1, descending=desc[1])]
    check(ctx, [P.INT8, P.INT8], [hi, lo], keys, [1, 64, 100, 65537, n])


# --- NULLs -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("density", ["none", "sparse", "dense", "all"])
def test_null_maps(ctx, density, desc):
    n = 250000
    rng = np.random.default_rng(5)
    frac = {"none": 0.0, "sparse": 0.001, "dense": 0.7, "all": 1.0}[density]
    null = (rng.random(n) < frac).astype(np.uint8)
    cols = [rng.integers(-1000, 1000, n), rng.integers(-10**6, 10**6, n)]
    keys = [dict(col=0, descending=desc, nulls=MAP), dict(col=1, descending=1 - desc)]
    check(ctx, [P.INT8, P.INT8], cols, keys, [1, 64, 65, 100, 4096, n - 1, n], nulls=[null, None])


@pytest.mark.parametrize("desc", [0, 1])
def test_count_column_null_source(ctx, desc):
    """a sum state: N = 0 makes (hi, lo) NULL whatever they hold"""
    n = 120000
    rng = np.random.default_rng(8)
    cnt = rng.integers(0, 4, n)
    hi = rng.integers(-1, 1, n, endpoint=True)
    lo = rng.integers(-2**63, 2**63 - 1, n, endpoint=True)
    keys = [dict(col=1, descending=desc, nulls=COUNT, null_col=0), dict(col=2, unsigned_cmp=1, descending=desc, nulls=COUNT,
                                                                        null_col=0)]
    check(ctx, [P.INT8, P.INT8, P.INT8], [cnt, hi, lo], keys, [1, 100, 65537, n])


# --- float8 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("desc", [0, 1])
def test_float8_specials(ctx, desc):
    n = 300000
    rng = np.random.default_rng(12)
    f = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5, 5e-324, -5e-324, 1e308, -1e308]), n)
    mixed = rng.random(n) < 0.3
    f[mixed] = rng.standard_normal(int(mixed.sum()))
    bits = f.view(np.int64).copy()
    nan_rows = rng.random(n) < 0.05
    payloads = np.array([0x7FF8000000000000, 0x7FF0000000000001, -0x0008000000000000, 0x7FFFFFFFFFFFFFFF], dtype=np.int64)
    bits[nan_rows] = rng.choice(payloads, int(nan_rows.sum()))
    null = (rng.random(n) < 0.02).astype(np.uint8)
    keys = [dict(col=0, float8=1, descending=desc, nulls=MAP), dict(col=1)]
    check(ctx, [P.FLOAT8, P.INT4], [bits.view(np.float64), rng.integers(0, 3, n).astype(np.int32)], keys,
          [1, 64, 65, 100, 4096, 65537, n], nulls=[null, None])


def test_float8_sum_bits_in_an_int8_column(ctx):
    """a float8 sum state's lo: float8 order over an int8 column"""
    n = 100000
    rng = np.random.default_rng(13)
    bits = (rng.standard_normal(n) * 1e3).view(np.int64)
    check(ctx, [P.INT8], [bits], [dict(col=0, float8=1, descending=1)], [1, 100, n])


# --- ties --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5000, 10**6])
def test_constant_and_tied_keys(ctx, n):
    """every row equal: rows 0 .. limit - 1, with no digit to count; then a key with three values and a tied second key"""
    cols = [np.full(n, 42, dtype=np.int64), np.arange(n) % 3, np.zeros(n, dtype=np.int32)]
    dev = upload(ctx, [P.INT8, P.INT8, P.INT4], cols)
    try:
        for limit in (1, 65, n):
            got, names = device(ctx, dev, [dict(col=0, descending=1), dict(col=2)], limit)
            assert got == list(range(min(limit, n))) and names == ["k_tsel_image", "k_tsel_finish"], (limit, names)
    finally:
        dev.free()
    check(ctx, [P.INT8, P.INT8, P.INT4], cols, [dict(col=1, descending=1), dict(col=0), dict(col=2)], [1, 65, 4096, n])


def test_refusals_name_the_problem(ctx):
    dev = upload(ctx, [P.INT4, P.FLOAT8], [np.zeros(10, dtype=np.int32), np.zeros(10)])
    try:
        for keys, frag in (([dict(col=0, float8=1)], "narrower than 8 bytes"),
                           ([dict(col=1, nulls=COUNT, null_col=0)], "not an int8 column"), ([dict(col=5)], "bad key column")):
            with pytest.raises(capi.CbgpuError) as e:
                capi.topn_select(ctx, dev, keys, 10)
            assert frag in str(e.value)
    finally:
        dev.free()


# --- through the executor ----------------------------------------------------------------------------------------------------
def _text(rows):
    return [tuple(map(str, r)) for r in rows]


def _nullable_fact(n, seed):
    """fact with NULLs in k and v, and every v NULL in the groups k % 5 == 0 (a NULL sum / min / max); x integer-valued, so
    float8 sums are exact in any order"""
    fo, fp = make(fact, n, seed=seed, null_frac=0.05)
    for rel in (fo, fp):
        k = rel.columns[0]
        rel.nulls[1][k % 5 == 0] = 1
        rel.columns[3][:] = np.round(rel.columns[3] - 500.0)
    return fo, fp


ORDERS = {
    # (group keys, aggregates, sort keys [(attno, descending)]): every order ends in the unique group key, so it is total
    "k": (["k"], [("n", P.AGG_COUNT_STAR, None)], [(1, False)]),
    "k_desc": (["k"], [("n", P.AGG_COUNT_STAR, None)], [(1, True)]),
    "sum_v": (["k"], [("s", P.AGG_SUM, "v")], [(2, False), (1, False)]),
    "sum_v_desc": (["k"], [("s", P.AGG_SUM, "v")], [(2, True), (1, False)]),
    "min_v": (["k"], [("m", P.AGG_MIN, "v")], [(2, False), (1, True)]),
    "max_v_desc": (["k"], [("m", P.AGG_MAX, "v")], [(2, True), (1, False)]),
    "sum_x": (["k"], [("s", P.AGG_SUM, "x")], [(2, False), (1, False)]),
    "max_x_desc": (["k"], [("m", P.AGG_MAX, "x")], [(2, True), (1, True)]),
}


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("order", list(ORDERS))
def test_limit_sort_over_nullable_and_float8_keys(ctx, oracle, order, generic, mem_kb):
    fo, fp = _nullable_fact(60000, seed=21)
    names = ["k", "v", "amt", "x", "g"]
    gkeys, aggs, sort_keys = ORDERS[order]
    agg = agg_over(scan(1, fo, names), names, gkeys, aggs)
    for limit in (1, 10, 64, 65, 100, 5000):
        dev = to_device(ctx, [fp])
        ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
        plan = P.LimitSort(agg, sort_keys, limit)
        ctx.trace_begin()
        try:
            got = ex.run(plan).rows
        finally:
            trace = [x for x, _ in ctx.trace_end() if x.startswith(("k_topn", "k_tsel"))]
            ex.close()
            for d in dev:
                d.free()
        want = oracle.execute(plan, [[fo]]).rows
        assert _text(got) == _text(want), (order, limit, got[:4], want[:4])
        assert trace and all(x.startswith("k_tsel") for x in trace), trace


def test_all_null_sum_sorts_as_null(ctx, oracle):
    """ORDER BY sum(v) over groups whose v are all NULL: the sums are NULL, last ascending and first descending - not 0"""
    fo, fp = _nullable_fact(2000, seed=22)
    names = ["k", "v"]
    agg = agg_over(scan(1, fo, names), names, ["k"], [("s", P.AGG_SUM, "v")])
    for desc in (False, True):
        got, want = run_both(ctx, oracle, P.LimitSort(agg, [(2, desc), (1, False)], 12), [fo], [fp], False)
        assert _text(got) == _text(want), (desc, got, want)
        assert any(r[1] is None for r in want) == desc


def test_left_join_column(ctx, oracle):
    """ORDER BY a column of the NULL-extended side of a LEFT join (w), then the outer key"""
    fo, fp = make(fact, 20000, seed=23)
    do, dp = make(dim, 20, seed=24, kmax=50)
    sf = scan(1, fo, ["k", "amt"])
    sd = scan(2, do, ["dk", "w", "c"])
    h = P.Hash(sd, [P.out_var(sd, 1)])
    targets = [("k", P.out_var(sf, 1)), ("w", P.InnerVar(2, P.INT8))]
    j = P.HashJoin(P.JOIN_LEFT, sf, h, [P.out_var(sf, 1)], targets)
    agg = agg_over(j, ["k", "w"], ["w", "k"], [("n", P.AGG_COUNT_STAR, None)])
    for keys in ([(1, False), (2, False)], [(1, True), (2, True)]):
        for limit in (5, 40, 100):
            got, want = run_both(ctx, oracle, P.LimitSort(agg, keys, limit), [fo, do], [fp, dp], False)
            assert _text(got) == _text(want), (keys, limit, got[:4], want[:4])


# --- TPC-H Q21 at its own LIMIT 100 ------------------------------------------------------------------------------------------
def _run_q21(ctx, sf, generic=False, mem_kb=0):
    dev = to_device(ctx, tpch_q21.gen_tables(sf, capi.hashbpchar))
    ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
    try:
        return [tuple(r) for r in ex.run(tpch_q21.q21_plan(limit=100)).rows]
    finally:
        ex.close()
        for d in dev:
            d.free()


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("generic", [False, True])
def test_q21_limit_100_sf001_against_the_oracle(ctx, oracle, generic, mem_kb):
    want = [tuple(r) for r in oracle.execute(tpch_q21.q21_plan(limit=100), [tpch_q21.gen_tables(0.01, oracle.hashbpchar)]).rows]
    assert _run_q21(ctx, 0.01, generic, mem_kb) == want and len(want) >= 1


def test_q21_limit_100_sf1_against_numpy(ctx):
    want = tpch_q21.numpy_answer(1, limit=100)
    assert _run_q21(ctx, 1) == want and len(want) == 100
