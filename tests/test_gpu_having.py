"""HAVING on the device (cbgpu_having_select, k_having_eval / k_having_scan / k_having_scatter).

- The entry point against the Python reference of tests/having_ref.py: random programs over random groups relations of 0 to
  2^22 + 5 groups; the selection must be the reference's ascending id list, element for element.
- Through the executor against Python: count / sum / avg / min / max with NULL states, numeric keys and constants of different
  scales, AGG_PLAIN, float8 min / max / sum / avg and float8 keys with NaN and -0, on both kernel routes and under a 16 KB
  budget; Q18 on three segments and at SF1 against numpy.
- A cross-product beyond 128 bits is CBGPU_ERR_OVERFLOW, and the executor runs again afterwards.
- A dictionary-coded grouping column in HAVING is refused before any launch: the host evaluator this replaces compared its
  dictionary codes with the constant's value."""
import math
import random
from collections import defaultdict
from decimal import Decimal

import numpy as np
import pytest

import having_ref as H
from cloudberry_b200 import capi, tpch_q10_q18 as Q
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import shard, to_device

pytestmark = pytest.mark.gpu
OVERFLOW, UNSUPPORTED = -4, -3
HAVING_KERNELS = ("k_having_eval", "k_having_scan", "k_having_scatter")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


# ---- the entry point ----
def groups_relation(n, rng):
    """keys k_int (int4, NULLs), k_num (numeric, scale 2), k_f8 (float8 with NaN / -0 / inf), k_ch (character(1)); then three
    accumulators' (N, lo, hi): an exact one, a float8 sum, a float8 min (F8ORD images)"""
    nrng = np.random.default_rng(rng.randint(0, 2**31))
    k_int = nrng.integers(-1000, 1000, n, dtype=np.int32)
    k_int_null = (nrng.random(n) < 0.05).astype(np.uint8)
    k_num = nrng.integers(-10**6, 10**6, n, dtype=np.int64)
    specials = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 0.5, -0.5], dtype=np.float64)
    k_f8 = np.where(nrng.random(n) < 0.2, specials[nrng.integers(0, len(specials), n)], nrng.integers(-40, 40, n) / 4.0)
    k_ch = nrng.integers(32, 127, n, dtype=np.uint8)
    n0 = np.where(nrng.random(n) < 0.1, 0, nrng.integers(1, 50, n)).astype(np.int64)
    lo0 = nrng.integers(-10**9, 10**9, n, dtype=np.int64)
    hi0 = np.where(lo0 < 0, -1, 0).astype(np.int64)
    n1 = np.where(nrng.random(n) < 0.1, 0, nrng.integers(1, 50, n)).astype(np.int64)
    s1 = np.where(nrng.random(n) < 0.05, specials[nrng.integers(0, len(specials), n)], nrng.integers(-400, 400, n) / 8.0)
    n2 = n1.copy()
    m2 = np.array([H.f8ord(int(b)) for b in s1[::-1].view(np.int64)], dtype=np.int64) if n else np.zeros(0, np.int64)
    cols = [k_int, k_num, k_f8.view(np.int64), k_ch, n0, lo0, hi0, n1, s1.view(np.int64), np.zeros(n, np.int64),
            n2, m2, np.zeros(n, np.int64)]
    types = [P.INT4, P.NUMERIC, P.FLOAT8, P.BPCHAR1] + [P.INT8] * 9
    host = HostRelation("groups", ["c%d" % i for i in range(len(cols))], types,
                        [k_f8 if t == P.FLOAT8 else c for c, t in zip(cols, types)], nulls=[k_int_null] + [None] * 12)
    widths = [4, 8, 8, 1] + [8] * 9
    ref = [(w, c, k_int_null if i == 0 else None, i == 2) for i, (w, c) in enumerate(zip(widths, cols))]
    return host, ref


def random_program(rng):
    """compares of the relation's keys, constants and states under AND / OR / NOT; 1 to 3 quals"""
    def leaf(f8):
        r = rng.random()
        if r < 0.3:
            return [(H.CBP_LOAD, 2, 0)] if f8 else [rng.choice([(H.CBP_LOAD, 0, rng.randint(0, 3)), (H.CBP_LOAD, 1, 2),
                                                                (H.CBP_LOAD, 3, 0)])]
        if r < 0.6:
            if f8:
                return [(H.CBP_CONST, H.CBH_CONST_F8, H.f8_bits(rng.choice([0.0, -0.0, 1.0, -2.5, 0.125, math.nan, math.inf])))]
            return [(H.CBP_CONST, rng.randint(0, 18), rng.randint(-10**6, 10**6) * 10 ** rng.randint(0, 12))]
        if f8:
            return [rng.choice([(H.CBP_STATE, 7, H.CBH_FSUM), (H.CBP_STATE, 7, H.CBH_FAVG), (H.CBP_STATE, 10, H.CBH_FMIN)])]
        return [(H.CBP_STATE, 4, rng.choice([H.CBH_COUNT, H.CBH_SUM, H.CBH_AVG, H.CBH_MIN, H.CBH_MAX]) | rng.randint(0, 4) << 8)]

    def boolean(depth):
        r = rng.random()
        if depth == 0 or r < 0.5:
            f8 = rng.random() < 0.4
            return leaf(f8) + leaf(f8) + [((H.CBP_FEQ if f8 else H.CBP_EQ) + rng.randint(0, 5), 0, 0)]
        if r < 0.65:
            return boolean(depth - 1) + [(H.CBP_NOT, 0, 0)]
        op = H.CBP_AND if rng.random() < 0.5 else H.CBP_OR
        return boolean(depth - 1) + boolean(depth - 1) + [(op, 0, 0)]

    nq = rng.randint(1, 3)
    return [o for _ in range(nq) for o in boolean(2)], nq


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 65537])
def test_entry_point_matches_reference(ctx, n):
    rng = random.Random(n + 7)
    host, ref = groups_relation(n, rng)
    dev = capi.DeviceRelation.from_host(ctx, host)
    try:
        for _ in range(3 if n > 1000 else 8):
            ops, nq = random_program(rng)
            want = [g for g in range(n) if H.keep(ops, ref, g, nq)[0]]
            got = capi.having_select(ctx, dev, ops, nq)
            assert got.tolist() == want, ops
    finally:
        dev.free()


def test_entry_point_at_four_million_groups(ctx):
    """2^22 + 5 groups: sum(x) > 50 (x of scale 2) AND k_int <= 100 (NULL keys fail), checked with numpy"""
    n = (1 << 22) + 5
    host, ref = groups_relation(n, random.Random(5))
    dev = capi.DeviceRelation.from_host(ctx, host)
    try:
        ops = [(H.CBP_STATE, 4, H.CBH_SUM | 2 << 8), (H.CBP_CONST, 0, 50), (capi.CBP_GT, 0, 0),
               (H.CBP_LOAD, 0, 0), (H.CBP_CONST, 0, 100), (capi.CBP_LE, 0, 0)]
        got = capi.having_select(ctx, dev, ops, 2)
        _, k_int, null, _ = ref[0]
        want = np.nonzero((ref[4][1] != 0) & (ref[5][1] > 5000) & (null == 0) & (k_int <= 100))[0]
        assert len(want) > 100000 and np.array_equal(got, want.astype(np.uint32))
    finally:
        dev.free()


def test_entry_point_overflow_then_runs_again(ctx):
    rng = random.Random(3)
    host, _ = groups_relation(1000, rng)
    dev = capi.DeviceRelation.from_host(ctx, host)
    try:
        # avg of scale 0 against a constant of scale 1000: the constant's side is scaled by 10^1000
        with pytest.raises(capi.CbgpuError) as e:
            capi.having_select(ctx, dev, [(H.CBP_STATE, 4, H.CBH_AVG), (H.CBP_CONST, 1000, 1), (capi.CBP_GT, 0, 0)], 1)
        assert e.value.code == OVERFLOW
        assert len(capi.having_select(ctx, dev, [(H.CBP_STATE, 4, H.CBH_COUNT), (H.CBP_CONST, 0, 0), (capi.CBP_GE, 0, 0)], 1)) == 1000
    finally:
        dev.free()


def test_entry_point_refuses_malformed_programs_before_any_launch(ctx):
    host, _ = groups_relation(100, random.Random(4))
    dev = capi.DeviceRelation.from_host(ctx, host)
    bad = [([(H.CBP_STATE, 4, H.CBH_SUM), (H.CBP_CONST, H.CBH_CONST_F8, 0), (capi.CBP_GT, 0, 0)], 1, "two exact or two float8"),
           ([(H.CBP_LOAD, 0, 0), (H.CBP_CONST, 0, 1), (capi.CBP_ADD, 0, 0)], 1, "opcode not supported"),
           ([(H.CBP_LOAD, 0, 0), (H.CBP_CONST, 0, 1), (capi.CBP_GT, 0, 0)], 2, "not one per qual"),
           ([(H.CBP_STATE, 2, H.CBH_SUM), (H.CBP_CONST, 0, 1), (capi.CBP_GT, 0, 0)], 1, "not (N, lo, hi)")]
    try:
        for ops, nq, msg in bad:
            before = ctx.launches()
            with pytest.raises(capi.CbgpuError) as e:
                capi.having_select(ctx, dev, ops, nq)
            assert e.value.code == -2 and msg in str(e.value) and ctx.launches() == before, (ops, str(e.value))
    finally:
        dev.free()


# ---- through the executor ----
NROWS = 20000


def fact_table():
    """g (int4 key, NULLs; groups 490.. have only NULL x), d (numeric(.., 1) key), fk (float8 key with NaN), x (numeric,
    scale 2, NULLs), f (float8 multiples of 1/4, -0, NaN in group 7; group 3's least value is 0 or -0): float8 sums are exact
    in any order"""
    rng = np.random.default_rng(11)
    g = rng.integers(0, 500, NROWS).astype(np.int32)
    gnull = (rng.random(NROWS) < 0.02).astype(np.uint8)
    d = rng.integers(0, 60, NROWS).astype(np.int64)
    fk = rng.choice(np.array([np.nan, 0.0, 1.5, -2.0, np.inf, 3.25]), NROWS)
    x = rng.integers(-5000, 20000, NROWS).astype(np.int64)
    xnull = ((rng.random(NROWS) < 0.1) | (g >= 490)).astype(np.uint8)
    f = rng.integers(-40, 41, NROWS) / 4.0
    f[g == 3] = np.abs(f[g == 3])
    f[((g == 3) | (rng.random(NROWS) < 0.01)) & (rng.random(NROWS) < 0.3)] = -0.0
    f[(g == 7) & (rng.random(NROWS) < 0.5)] = np.nan
    return HostRelation("t", ["g", "d", "fk", "x", "f"], [P.INT4, P.NUMERIC, P.FLOAT8, P.NUMERIC, P.FLOAT8], [g, d, fk, x, f],
                        dscales=[0, 1, 0, 2, 0], nulls=[gnull, None, None, xnull, None])


def groups_of(t, key):
    """key value (None for NULL, 'nan' for NaN) -> rows"""
    out = defaultdict(list)
    kc = t.columns[t.names.index(key)]
    kn = t.nulls[t.names.index(key)]
    for i in range(t.nrows):
        k = None if kn is not None and kn[i] else kc[i].item()
        out["nan" if isinstance(k, float) and math.isnan(k) else k].append(i)
    return out


def canon(v):
    if v is None:
        return (0, "")
    if isinstance(v, float):
        return (1, "nan") if math.isnan(v) else (2, repr(v + 0.0))
    return (3, str(Decimal(str(v)).normalize()))


def scan_t(t):
    return P.SeqScan(1, [(n, P.Var(1, i + 1, t.types[i], t.dscales[i])) for i, n in enumerate(t.names)])


def v(sc, name, t):
    i = t.names.index(name)
    return P.out_var(sc, i + 1)


def agg_plan(t, key, quals):
    sc = scan_t(t)
    keys = [t.names.index(key) + 1] if key else []
    targets = ([(key, v(sc, key, t))] if key else []) + [("n", P.Aggref(P.AGG_COUNT_STAR))]
    return P.Agg(sc, P.AGG_HASHED if key else P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, keys, targets, num_groups=600,
                 quals=[q(sc) for q in quals])


def cases(t):
    """(key, quals, Python predicate over (key value, x values (None = NULL), f values))"""
    X, F = lambda sc: v(sc, "x", t), lambda sc: v(sc, "f", t)
    nums = lambda xs: [Decimal(a) / 100 for a in xs if a is not None]     # noqa: E731
    return [
        ("g", [lambda sc: P.OpExpr(P.OP_GE, P.Aggref(P.AGG_COUNT_STAR), P.Const(P.INT8, 40)),
               lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_SUM, X(sc)), P.NumericConst("2500.5"))],
         lambda k, xs, fs: len(xs) >= 40 and bool(nums(xs)) and sum(nums(xs)) > Decimal("2500.5")),
        ("g", [lambda sc: P.BoolExpr(P.OR_EXPR,
                                     P.OpExpr(P.OP_LE, P.Aggref(P.AGG_AVG, X(sc)), P.NumericConst("60.125")),
                                     P.BoolExpr(P.NOT_EXPR, P.OpExpr(P.OP_LT, P.Aggref(P.AGG_MAX, X(sc)), P.NumericConst("199.9")))),
               lambda sc: P.OpExpr(P.OP_NE, P.Aggref(P.AGG_COUNT, X(sc)), P.Const(P.INT8, 0))],
         lambda k, xs, fs: bool(nums(xs)) and (sum(nums(xs)) / len(nums(xs)) <= Decimal("60.125") or max(nums(xs)) >= Decimal("199.9"))),
        ("g", [lambda sc: P.BoolExpr(P.OR_EXPR, P.OpExpr(P.OP_LT, P.Aggref(P.AGG_MIN, X(sc)), P.NumericConst("-49")),
                                     P.OpExpr(P.OP_GT, v(sc, "g", t), P.Const(P.INT4, 480)))],
         lambda k, xs, fs: (k is not None and k > 480) or (bool(nums(xs)) and min(nums(xs)) < -49)),
        ("d", [lambda sc: P.OpExpr(P.OP_GE, v(sc, "d", t), P.NumericConst("2.500")),
               lambda sc: P.OpExpr(P.OP_LT, P.Aggref(P.AGG_SUM, X(sc)), P.NumericConst("24000.5"))],
         lambda k, xs, fs: Decimal(k) / 10 >= Decimal("2.5") and bool(nums(xs)) and sum(nums(xs)) < Decimal("24000.5")),
        ("g", [lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_MAX, F(sc)), P.Const(P.FLOAT8, 9.5)),
               lambda sc: P.OpExpr(P.OP_LE, P.Aggref(P.AGG_SUM, F(sc)), P.Const(P.FLOAT8, 40.125))],
         lambda k, xs, fs: _f8max(fs) > 9.5 and _f8le(math.fsum(fs) if not any(map(math.isnan, fs)) else math.nan, 40.125)),
        ("g", [lambda sc: P.OpExpr(P.OP_EQ, P.Aggref(P.AGG_MIN, F(sc)), P.Const(P.FLOAT8, 0.0)),
               lambda sc: P.OpExpr(P.OP_GE, P.Aggref(P.AGG_AVG, F(sc)), P.Const(P.FLOAT8, -0.0))],
         lambda k, xs, fs: min(fs, key=lambda a: (math.isnan(a), a)) == 0.0 and not _f8lt(sum(fs) / len(fs), 0.0)),
        ("g", [lambda sc: P.OpExpr(P.OP_LE, P.Aggref(P.AGG_MIN, F(sc)), P.Const(P.FLOAT8, -9.5)),
               lambda sc: P.OpExpr(P.OP_LT, P.Aggref(P.AGG_AVG, F(sc)), P.Const(P.FLOAT8, 0.0625))],
         lambda k, xs, fs: _f8le(min(fs, key=lambda a: (math.isnan(a), a)), -9.5) and _f8lt(sum(fs) / len(fs), 0.0625)),
        ("fk", [lambda sc: P.OpExpr(P.OP_GE, v(sc, "fk", t), P.Const(P.FLOAT8, 0.0)),
                lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_AVG, F(sc)), P.Const(P.FLOAT8, -0.0625))],
         lambda k, xs, fs: (k == "nan" or k >= 0.0) and not _f8le(sum(fs) / len(fs), -0.0625)),
    ]


def _f8lt(a, b):        # float8_cmp_internal: NaN above everything
    return False if math.isnan(a) else True if math.isnan(b) else a < b


def _f8le(a, b):
    return not _f8lt(b, a)


def _f8max(fs):
    return max(fs, key=lambda a: (math.isnan(a), a))


def expected(t, key, pred):
    x, xn, f = t.columns[3], t.nulls[3], t.columns[4]
    out = []
    for k, rows in (groups_of(t, key).items() if key else [(None, list(range(t.nrows)))]):
        xs = [None if xn[i] else int(x[i]) for i in rows]
        fs = [float(f[i]) for i in rows]
        if pred(k, xs, fs):
            k = Decimal(k) / 10 if key == "d" else math.nan if k == "nan" else k
            out.append((canon(k), len(rows)) if key else len(rows))
    return sorted(out)


@pytest.fixture(scope="module")
def fact(ctx):
    t = fact_table()
    d = capi.DeviceRelation.from_host(ctx, t)
    yield t, d
    d.free()


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("generic", [False, True])
def test_executor_having_against_python(ctx, fact, generic, mem_kb):
    t, d = fact
    ex = capi.Executor(ctx, [d], force_generic=generic, operator_mem_kb=mem_kb)
    try:
        for i, (key, quals, pred) in enumerate(cases(t)):
            ctx.trace_begin()
            rows = ex.run(agg_plan(t, key, quals)).rows
            names = [n for n, _ in ctx.trace_end()]
            want = expected(t, key, pred)
            assert 0 < len(want) < len(groups_of(t, key)), i
            assert sorted((canon(r[0]), int(r[1])) for r in rows) == want, i
            assert all(k in names for k in HAVING_KERNELS), names
    finally:
        ex.close()


def test_executor_plain_aggregate(ctx, fact):
    t, d = fact
    ex = capi.Executor(ctx, [d])
    try:
        keep = ex.run(agg_plan(t, None, [lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_COUNT_STAR), P.Const(P.INT8, 5))])).rows
        drop = ex.run(agg_plan(t, None, [lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_SUM, v(sc, "x", t)),
                                                                       P.NumericConst("1000000000"))])).rows
        assert [int(r[0]) for r in keep] == [NROWS] and drop == []
    finally:
        ex.close()


def test_executor_overflow_then_runs_again(ctx, fact):
    """sum(x) of scale 2 against a constant of scale 38: the sum's side is scaled by 10^36, beyond 128 bits"""
    t, d = fact
    ex = capi.Executor(ctx, [d])
    try:
        tiny = "0." + "0" * 37 + "1"
        with pytest.raises(capi.CbgpuError) as e:
            ex.run(agg_plan(t, "g", [lambda sc: P.OpExpr(P.OP_GT, P.Aggref(P.AGG_SUM, v(sc, "x", t)), P.NumericConst(tiny))]))
        assert e.value.code == OVERFLOW
        key, quals, pred = cases(t)[0]
        assert sorted((canon(r[0]), int(r[1])) for r in ex.run(agg_plan(t, key, quals)).rows) == expected(t, key, pred)
    finally:
        ex.close()


def test_dictionary_key_is_refused_before_any_launch(ctx):
    """c_name compared with a constant of its own type: refused with no launch (a dictionary code says nothing of the order or
    the identity of strings across dictionaries)"""
    rels = Q.gen_tables(0.01, capi.hashbpchar)
    cust = [r for r in rels if r.name == "customer"][0]
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev)
    try:
        relid = [r.name for r in rels].index("customer") + 1
        i = cust.names.index("c_name")
        sc = P.SeqScan(relid, [("c_name", P.Var(relid, i + 1, cust.types[i], cust.dscales[i]))])
        plan = P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("c_name", P.out_var(sc, 1))], num_groups=1000,
                     quals=[P.OpExpr(P.OP_EQ, P.out_var(sc, 1), P.Const(cust.types[i], 0))])
        before = ctx.launches()
        with pytest.raises(capi.CbgpuError) as e:
            ex.run(plan)
        assert e.value.code == UNSUPPORTED and "dictionary-coded grouping column" in str(e.value)
        assert ctx.launches() == before
    finally:
        ex.close()
        for r in dev:
            r.free()


@pytest.mark.parametrize("threshold", [150, 212])
def test_q18_on_three_segments(ctx, oracle, threshold):
    """thresholds at which the subquery's HAVING keeps some orders and drops others on every segment"""
    rels = Q.gen_tables(0.01, capi.hashbpchar)
    segs = shard(oracle, rels, 3, Q.DIST_KEY)
    devs = [to_device(ctx, s) for s in segs]
    cl = capi.Cluster(ctx, devs)
    try:
        got = [tuple(r) for r in cl.run(Q.q18_plan(threshold=threshold, nsegs=3, sf=0.01)).rows]
    finally:
        cl.close()
        for dv in devs:
            for r in dv:
                r.free()
    want = Q.q18_numpy_answer(0.01, threshold=threshold)
    assert got == want and len(want) >= 3


def test_q18_sf1_against_numpy(ctx):
    rels = Q.gen_tables(1, capi.hashbpchar)
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev)
    try:
        ctx.trace_begin()
        res = ex.run(Q.q18_plan(sf=1))
        names = [n for n, _ in ctx.trace_end()]
    finally:
        ex.close()
        for r in dev:
            r.free()
    want = Q.q18_numpy_answer(1)
    assert [tuple(r) for r in res.rows] == want and len(want) >= 1
    assert all(names.count(k) == 1 for k in HAVING_KERNELS), names
    assert sum(v["having_ms"] for v in res.instrument.values()) > 0
