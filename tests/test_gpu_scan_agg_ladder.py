"""k_scan_agg_small, rung by rung, against the CPU oracle (-m gpu).

The fused scan -> qual -> few-group aggregate is not one kernel but a ladder: (4 groups, 32-bit multiply-accumulate)
-> (4 groups, 64-bit) on a failed overflow audit -> (8 groups, 64-bit) when one CTA sees more than 4 keys -> off the
ladder (k_probe_chain's aggregate sink, or the generic interpreter).  Each rung is instantiated per sum mask (0x10, 0x37, 0x3f) and input shape (1: qual + two keys,
2: qual and no key, 0: anything else), and the host picks among them from data-dependent audits.  Every case here
compares the oracle's rows exactly and also asserts which kernel finished the query (ctx.last_kernel(), the name
SA_LAUNCH gives it), so a case cannot pass by landing on another rung.

The plans are Agg(SeqScan) over non-null numeric(.,2) columns a, b, c, d with the product terms b*(k-c) and
b*(k-c)*(k2+d) of TPC-H Q1, grouped by a char(1) key and a dictionary key."""
from decimal import Decimal

import numpy as np
import pytest

from cloudberry_b200 import capi, tpch
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import canon, to_device

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
SA_TILE = 896                   # rows per pipeline stage of k_scan_agg_small (scan_agg.cu)
SA_NCONS4 = 448                 # consumer threads of the 4-group kernel: each takes rows ct and ct + 448 of a tile
GENERIC = "k_pipeline_generic"
# where a plan goes once the ladder gives up: k_probe_chain's aggregate sink takes up to two distinct sum terms (b*(k-c) alone
# here), the generic interpreter everything else
CHAIN = "k_probe_chain"


def small(g, mask, narrow, shape):
    return "k_scan_agg_small<%d,0x%x,%s,%d>" % (g, mask, "true" if narrow else "false", shape)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def table(n, seed=0, groups=4, vis=1.0, **cols):
    """n rows: keys k0 (char(1)) and k1 (dictionary, a function of k0, so (k0, k1) has `groups` values), an int4 qual
    column f and numeric columns a, b, c, d (scaled by 100).  Keyword arguments replace a column's values."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, groups, n)
    base = {
        "k0": (P.BPCHAR1, (ord("A") + g).astype(np.uint8)),
        "k1": (P.DICT8, (g % 3).astype(np.uint8)),
        "f": (P.INT4, rng.integers(-1000, 1000, n).astype(np.int32)),
        "a": (P.NUMERIC, rng.integers(100, 5001, n)),
        "b": (P.NUMERIC, rng.integers(90000, 10 ** 7, n)),
        "c": (P.NUMERIC, rng.integers(0, 11, n)),
        "d": (P.NUMERIC, rng.integers(0, 9, n)),
    }
    for k, v in cols.items():
        base[k] = (base[k][0], np.asarray(v(rng, n) if callable(v) else v).astype(base[k][1].dtype))
    names = list(base)
    visimap = None
    if vis < 1.0:
        visimap = np.packbits((rng.random(n) < vis).astype(np.uint8), bitorder="little")

    def rel():
        return HostRelation("t", names, [base[k][0] for k in names], [base[k][1] for k in names], visimap=visimap,
                            dict_texts=[["x0", "x1", "x2"] if k == "k1" else None for k in names])
    from oracle import oracle as O
    return rel().set_dict_hashes(O.hashbpchar), rel().set_dict_hashes(capi.hashbpchar)


def num(s):
    return P.NumericConst(s)


def rev(v, k="1.00"):
    return P.OpExpr(P.OP_MUL, v("b"), P.OpExpr(P.OP_SUB, num(k), v("c")))


def chg(v, k="1.00", k2="1.00"):
    return P.OpExpr(P.OP_MUL, rev(v, k), P.OpExpr(P.OP_ADD, num(k2), v("d")))


# sum sets, by the mask k_scan_agg_small instantiates for them
SUMS_10 = lambda v, k="1.00", k2=None: [("rev", P.AGG_SUM, rev(v, k))]                                   # noqa: E731
SUMS_37 = lambda v, k="1.00", k2="1.00": [("sa", P.AGG_SUM, v("a")), ("sb", P.AGG_SUM, v("b")),          # noqa: E731
                                          ("rev", P.AGG_SUM, rev(v, k)), ("chg", P.AGG_SUM, chg(v, k, k2)),
                                          ("avc", P.AGG_AVG, v("c"))]
SUMS_3F = lambda v, k="1.00", k2=None: [("sa", P.AGG_SUM, v("a")), ("sd", P.AGG_SUM, v("d")),            # noqa: E731
                                        ("rev", P.AGG_SUM, rev(v, k)), ("avb", P.AGG_AVG, v("b"))]


def plan_of(rel, keys=("k0", "k1"), sums=SUMS_37, qual=None, k="1.00", k2="1.00"):
    """Agg(SeqScan t): group by `keys`, qual (op, int32 constant) on f, the sums plus count(*)"""
    names = list(keys) + ["a", "b", "c", "d"]
    quals = [] if qual is None else [P.OpExpr(qual[0], P.Var(1, rel.attno("f"), P.INT4), P.Const(P.INT4, qual[1]))]
    tl = []
    for nme in names:
        a, t, ds = rel.var(nme)
        tl.append((nme, P.Var(1, a, t, ds)))
    sc = P.SeqScan(1, tl, quals)
    v = tpch._child_var(sc)
    aggs = sums(v, k, k2) + [("n", P.AGG_COUNT_STAR, None)]
    targets = [(kk, v(kk)) for kk in keys] + [(nme, P.Aggref(op, arg)) for nme, op, arg in aggs]
    strategy = P.AGG_HASHED if keys else P.AGG_PLAIN
    return P.Agg(sc, strategy, P.AGGSPLIT_SIMPLE, list(range(1, len(keys) + 1)), targets, num_groups=64)


def _scaled_diff(got, want):
    """per row and column, (got - want) in units of 2^32 of the column's last digit, where they differ"""
    out = []
    for g, w in zip(canon(got), canon(want)):
        for x, y in zip(g, w):
            if x != y and isinstance(x, str) and isinstance(y, str):
                d = Decimal(x) - Decimal(y)
                out.append(str(d.scaleb(-d.as_tuple().exponent) / 2 ** 32 if d else 0))
    return out


def run(ctx, oracle, rels, plan, kernel):
    fo, fp = rels
    dev = to_device(ctx, [fp])
    ex = capi.Executor(ctx, dev)
    try:
        got = ex.run(plan).rows
        name = ctx.last_kernel()[0]
    finally:
        ex.close()
        for d in dev:
            d.free()
    want = oracle.execute(plan, [[fo]]).rows
    assert canon(got) == canon(want), ("differences in 2^32 units of the last digit", _scaled_diff(got, want))
    assert name == kernel
    return want


# ---- sign: b*(k-c) may be negative; the 32-bit form must then be refused ----

@pytest.mark.parametrize("shape", [1, 2, 0])
def test_negative_rev_some_rows(ctx, oracle, shape):
    """sum(b*(1.00-c)) with c > 1.00 on about half the rows: each such product is negative.  b < 2^23 and c < 2^8 keep the
    bit-count bound of b*(k-c) at 32, so only the sign can refuse the 32-bit form"""
    rels = table(20011, seed=1, b=lambda rng, n: rng.integers(0, 2 ** 23, n), c=lambda rng, n: rng.integers(0, 201, n))
    keys = {1: ("k0", "k1"), 2: (), 0: ("k0",)}[shape]
    qual = None if shape == 0 else (P.OP_LE, 900)
    run(ctx, oracle, rels, plan_of(rels[0], keys, SUMS_10, qual), small(4, 0x10, False, shape))


@pytest.mark.parametrize("k", ["0.00", "-1.00", "-0.01"])
def test_rev_with_zero_or_negative_k(ctx, oracle, k):
    """sum(b*(k-c)) with k = 0 or k < 0: every product with c > 0 is negative"""
    rels = table(5003, seed=2)
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_GE, -500), k=k), small(4, 0x37, False, 1))
    assert all(r[4].startswith("-") for r in want)


def test_negative_k2_plus_d_keeps_narrow(ctx, oracle):
    """b*(k-c)*(k2+d) with k2+d < 0 on most rows: that sum is always 64-bit, b*(k-c) >= 0, so the 32-bit rung stays"""
    rels = table(7001, seed=3)
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_LT, 700), k2="-5.00"), small(4, 0x37, True, 1))
    assert all(r[5].startswith("-") for r in want)


def test_negative_rev_and_negative_k2_plus_d(ctx, oracle):
    """both factors change sign row by row: products of either sign in both sums"""
    rels = table(7001, seed=4, c=lambda rng, n: rng.integers(0, 300, n), d=lambda rng, n: rng.integers(0, 1000, n))
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_LT, 700), k="1.50", k2="-5.00"), small(4, 0x37, False, 1))


@pytest.mark.parametrize("col", ["a", "b", "c", "d"])
def test_negative_input_leaves_the_ladder(ctx, oracle, col):
    """a negative input breaks the bit-count bounds of both 64-bit and 32-bit rungs: the generic kernel answers"""
    def neg(rng, n):
        v = rng.integers(0, 1000, n)
        v[rng.integers(0, n, 5)] = -7
        return v
    rels = table(3001, seed=5, **{col: neg})
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_3F if col == "d" else SUMS_37, qual=(P.OP_GT, -900)), GENERIC)


# ---- the audit's boundaries ----

def _small_b(rng, n):
    return rng.integers(0, 1000, n)     # mask 0x3f also audits b*(k-c)*d: keep it far below 63 bits


def test_d_of_32_bits_keeps_narrow(ctx, oracle):
    """the 32-bit form sums d = 2^32 - 1 exactly (IMAD.WIDE.U32 of a full 32-bit operand)"""
    rels = table(4001, seed=6, b=_small_b, d=lambda rng, n: np.full(n, 2 ** 32 - 1))
    run(ctx, oracle, rels, plan_of(rels[0], keys=("k0",), sums=SUMS_3F), small(4, 0x3f, True, 0))


def test_d_of_33_bits_refuses_narrow(ctx, oracle):
    rels = table(4001, seed=6, b=_small_b, d=lambda rng, n: np.where(np.arange(n) == 17, 2 ** 32, 2 ** 32 - 1))
    run(ctx, oracle, rels, plan_of(rels[0], keys=("k0",), sums=SUMS_3F), small(4, 0x3f, False, 0))


@pytest.mark.parametrize("bbits,narrow", [(24, True), (25, False)])
def test_rev_of_32_bits(ctx, oracle, bbits, narrow):
    """b < 2^bbits, k = 1.00 (7 bits), c < 16: b*(k-c) has at most bbits + 8 bits; 32 keeps the 32-bit form"""
    rels = table(6007, seed=7, b=lambda rng, n: np.where(np.arange(n) == 5, 2 ** bbits - 1, rng.integers(0, 2 ** 20, n)),
                 c=lambda rng, n: rng.integers(0, 16, n))
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_10, qual=(P.OP_LE, INT32_MAX)), small(4, 0x10, narrow, 1))


@pytest.mark.parametrize("bbits,rung", [(40, small(4, 0x10, False, 2)), (41, CHAIN)])
def test_rev_near_2_62(ctx, oracle, bbits, rung):
    """b*(k-c) with k = 10000.00 (20 bits), c < 2^20: products up to 2^(bbits + 20), bounded by 2^61 / 2^62 with the sign
    bit's headroom.  One row per thread: 2^61 passes the 64-bit rung, 2^62 leaves the ladder.  Either way exact."""
    n = SA_NCONS4
    rels = table(n, seed=8, b=lambda rng, n: np.where(np.arange(n) == 0, 2 ** bbits - 1, 1),
                 c=lambda rng, n: rng.integers(0, 2 ** 20, n))
    run(ctx, oracle, rels, plan_of(rels[0], keys=(), sums=SUMS_10, qual=(P.OP_GE, INT32_MIN), k="10000.00"), rung)


@pytest.mark.parametrize("n,rung", [(SA_NCONS4, small(4, 0x10, False, 2)), (SA_NCONS4 + 1, CHAIN)])
def test_rows_per_thread_cross_63_bits(ctx, oracle, n, rung):
    """the same 61-bit product bound: one more row on thread 0 (rows 0 and 448 of the first tile) adds a bit to its
    partial-sum bound, 62 + 1 = 63 is refused"""
    rels = table(n, seed=9, b=lambda rng, n: np.where(np.arange(n) == 0, 2 ** 40 - 1, 1),
                 c=lambda rng, n: rng.integers(0, 2 ** 20, n))
    run(ctx, oracle, rels, plan_of(rels[0], keys=(), sums=SUMS_10, qual=(P.OP_GE, INT32_MIN), k="10000.00"), rung)


@pytest.mark.parametrize("tiles_per_cta,rung", [(7, small(4, 0x10, False, 0)), (8, CHAIN)])
def test_many_rows_per_thread_cross_63_bits(ctx, oracle, tiles_per_cta, rung):
    """the per-thread row count's bits over a table of many tiles per CTA.  Row 0 holds b = 2^37 - 1 (with k = 10000.00 and
    c < 2^20 a 58-bit product bound) on thread 0 of CTA 0, which sums 2 rows of each of its tiles: 7 full tiles and a
    partial one give it 15 rows, 58 + 4 bits pass; 8 full tiles give it 16 rows, 58 + 5 = 63 is refused"""
    n = ctx.sm_count() * SA_TILE * tiles_per_cta + (5 if tiles_per_cta == 7 else 0)
    rels = table(n, seed=10, groups=2, b=lambda rng, n: np.where(np.arange(n) == 0, 2 ** 37 - 1, 1),
                 c=lambda rng, n: rng.integers(0, 2 ** 20, n))
    run(ctx, oracle, rels, plan_of(rels[0], keys=("k0",), sums=SUMS_10, k="10000.00"), rung)


def test_product_beyond_64_bits_is_refused(ctx, oracle):
    rels = table(3001, seed=11, b=lambda rng, n: np.full(n, 4 * 10 ** 18), c=lambda rng, n: np.full(n, 4 * 10 ** 18))
    fo, fp = rels
    dev = to_device(ctx, [fp])
    ex = capi.Executor(ctx, dev)
    try:
        with pytest.raises(capi.CbgpuError):
            ex.run(plan_of(fp, sums=SUMS_10, qual=(P.OP_LE, 0), k="100.00"))
    finally:
        ex.close()
        for d in dev:
            d.free()


# ---- the ladder: groups per CTA, sum masks, shapes ----

@pytest.mark.parametrize("groups", [1, 2, 3, 4])
@pytest.mark.parametrize("sums,mask", [(SUMS_10, 0x10), (SUMS_37, 0x37), (SUMS_3F, 0x3f)])
def test_up_to_4_groups(ctx, oracle, groups, sums, mask):
    rels = table(50021, seed=20 + groups, groups=groups)
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=sums, qual=(P.OP_LT, 500)), small(4, mask, True, 1))
    assert len(want) == groups


@pytest.mark.parametrize("groups", [5, 8])
def test_5_to_8_groups_with_a_and_d(ctx, oracle, groups):
    """more than 4 keys in one CTA: the 8-group kernel (all six sums, 64-bit) needs columns a and d"""
    rels = table(50021, seed=30 + groups, groups=groups)
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_LT, 500)), small(8, 0x3f, False, 0))
    assert len(want) == groups


def test_5_to_8_groups_without_a_or_d(ctx, oracle):
    """without a and d the 8-group kernel cannot run: the ladder gives up"""
    rels = table(50021, seed=36, groups=6)
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_10, qual=(P.OP_LT, 500)), CHAIN)


@pytest.mark.parametrize("groups", [9, 40])
def test_9_or_more_groups(ctx, oracle, groups):
    rels = table(50021, seed=40 + groups, groups=groups)
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_LT, 500)), GENERIC)
    assert len(want) == groups


def test_groups_spread_over_ctas(ctx, oracle):
    """6 keys over the table, but each CTA's rows hold only 3 of them (one key per tile, tile t has key 2t / grid): the
    4-group rung stays, and the CTAs' partials for the same key are combined"""
    s = ctx.sm_count()
    n = s * SA_TILE * 3                                  # CTA b scans tiles b, b + s and b + 2s
    g = (np.arange(n) // SA_TILE) * 2 // s
    rels = table(n, seed=50, groups=6, k0=(ord("A") + g), k1=(g % 3))
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_GE, -900)), small(4, 0x37, True, 1))
    assert len(want) == 6


@pytest.mark.parametrize("shape,keys,qual", [(1, ("k0", "k1"), (P.OP_LE, 0)), (2, (), (P.OP_LE, 0)), (0, ("k0",), None),
                                             (0, ("k0", "k1"), None), (0, ("k1",), (P.OP_GT, 0))])
def test_shapes(ctx, oracle, shape, keys, qual):
    rels = table(30011, seed=60)
    run(ctx, oracle, rels, plan_of(rels[0], keys=keys, sums=SUMS_37, qual=qual), small(4, 0x37, True, shape))


# ---- quals, visibility, tiles ----

QUAL_EDGES = [(P.OP_EQ, INT32_MIN), (P.OP_EQ, INT32_MAX), (P.OP_LT, INT32_MAX), (P.OP_LE, INT32_MIN), (P.OP_LE, INT32_MAX),
              (P.OP_GT, INT32_MIN), (P.OP_GE, INT32_MIN), (P.OP_GE, INT32_MAX)]


@pytest.mark.parametrize("op,v", QUAL_EDGES)
def test_qual_at_int32_limits(ctx, oracle, op, v):
    """the qual folded to lo <= f <= lo + span at the ends of int32, with f = INT32_MIN / INT32_MAX on some rows"""
    def f(rng, n):
        x = rng.integers(-3, 4, n)
        x[rng.random(n) < 0.2] = INT32_MIN
        x[rng.random(n) < 0.2] = INT32_MAX
        return x
    rels = table(20011, seed=70, f=f)
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(op, v)), small(4, 0x37, True, 1))


@pytest.mark.parametrize("op,v", [(P.OP_LT, INT32_MIN), (P.OP_GT, INT32_MAX)])
def test_empty_qual_range(ctx, oracle, op, v):
    """f < INT32_MIN and f > INT32_MAX select nothing: the host hands the plan to the generic kernel"""
    rels = table(20011, seed=71, f=lambda rng, n: np.where(rng.random(n) < 0.5, INT32_MIN, INT32_MAX))
    want = run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(op, v)), GENERIC)
    assert want == []


@pytest.mark.parametrize("n", [1000, 100003])
@pytest.mark.parametrize("narrow", [True, False])
def test_visimap(ctx, oracle, n, narrow):
    """invisible rows are not aggregated, and their values do not reach the audit either way"""
    c = (lambda rng, n: rng.integers(0, 11, n)) if narrow else (lambda rng, n: rng.integers(0, 300, n))
    rels = table(n, seed=80, vis=0.7, c=c)
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_LE, 500)), small(4, 0x37, narrow, 1))


def _tile_counts():
    return [1, SA_NCONS4 - 1, SA_NCONS4, SA_NCONS4 + 1, SA_TILE - 1, SA_TILE, SA_TILE + 1, 2 * SA_TILE + 1]


@pytest.mark.parametrize("n", _tile_counts())
def test_rows_around_the_tile(ctx, oracle, n):
    rels = table(n, seed=90 + n % 97)
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_GE, -1000)), small(4, 0x37, True, 1))


@pytest.mark.parametrize("delta", [-1, 0, 1, SA_TILE + 1])
@pytest.mark.parametrize("waves", [1, 2])
def test_rows_around_the_grid(ctx, oracle, delta, waves):
    """grid x tile rows and its neighbours: the last CTA gets a partial tile, or one CTA gets one more tile"""
    n = waves * ctx.sm_count() * SA_TILE + delta
    rels = table(n, seed=100 + waves * 7 + delta % 13, c=lambda rng, n: rng.integers(0, 200, n))
    run(ctx, oracle, rels, plan_of(rels[0], sums=SUMS_37, qual=(P.OP_GE, -1000)), small(4, 0x37, False, 1))


# ---- Q1 keeps its kernel ----

def test_q1_golden_stays_narrow(ctx, oracle):
    rels, exp = tpch.load_golden(capi.hashbpchar)
    from oracle import oracle as O
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev)
    try:
        got = ex.run(tpch.q1_plan(1)).rows
        name = ctx.last_kernel()[0]
    finally:
        ex.close()
        for d in dev:
            d.free()
    assert tpch.format_q1(got) == tpch.format_q1(O.execute(tpch.q1_plan(1), [rels]).rows) == exp["q1"]
    assert name == small(4, 0x37, True, 1)


def test_q1_sf002_stays_narrow(ctx, oracle):
    rels_o = tpch.gen_tables(0.02, oracle.hashbpchar)
    rels_p = tpch.gen_tables(0.02, capi.hashbpchar)
    dev = to_device(ctx, rels_p)
    ex = capi.Executor(ctx, dev)
    try:
        got = ex.run(tpch.q1_plan(1)).rows
        name = ctx.last_kernel()[0]
    finally:
        ex.close()
        for d in dev:
            d.free()
    assert tpch.format_q1(got) == tpch.format_q1(oracle.execute(tpch.q1_plan(1), [rels_o]).rows)
    assert name == small(4, 0x37, True, 1)
