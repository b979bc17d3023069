"""LEFT, SEMI and ANTI hash joins with a join filter (joinqual) on the GPU (-m gpu): the pair probe tests the filter on every
key-equal candidate in its chain walk (cbgpu_ht_probe_pairs, k_ht_probe_filtered), SEMI / ANTI stop at the first
passing candidate, and a LEFT row none of whose candidates pass is NULL-extended once (nodeHashjoin.c:583-713).  Every query
is compared with the CPU oracle through both kernel routes, and the launch trace shows that the filtered probe ran.  Also:
the plan's own qual on non-inner joins, the same joins split into batches at a 16 KB operator budget, overflow inside the
filter, and direct calls to the C entry point against a numpy nested loop."""
import ctypes as C
import math

import numpy as np
import pytest

from cloudberry_b200 import capi
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import canon, to_device

pytestmark = pytest.mark.gpu

OVERFLOW = -4
TEXTS = ["t%d" % i for i in range(6)]
OUT_NAMES = ["k", "a", "f", "s", "e"]
IN_NAMES = ["ik", "b", "g", "t", "big"]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _nulls(rng, n, frac):
    return (rng.random(n) < frac).astype(np.uint8)


def _floats(rng, n):
    x = rng.integers(0, 40, n).astype(np.float64)
    x[rng.random(n) < 0.05] = np.nan
    return x


def outer_rel(n, seed, kmax):
    rng = np.random.default_rng(seed)
    cols = [rng.integers(0, kmax, n).astype(np.int32), rng.integers(0, 60, n), _floats(rng, n), rng.integers(0, 6, n).astype(np.uint8),
            np.full(n, 1 << 40, dtype=np.int64)]
    return HostRelation("o", OUT_NAMES, [P.INT4, P.INT8, P.FLOAT8, P.DICT8, P.INT8], cols,
                        nulls=[_nulls(rng, n, 0.1), _nulls(rng, n, 0.1), None, None, None], dict_texts=[None, None, None, TEXTS, None])


def inner_rel(n, seed, kmax, dup, unique_b=False, key_null=0.1):
    """dup: build rows per key (an int), or "skew": every build row has the same key"""
    rng = np.random.default_rng(seed)
    if dup == "skew":
        keys = np.full(n, 7, dtype=np.int32)
    else:
        keys = np.repeat(rng.permutation(kmax)[:max(n // dup, 0)], dup)[:n].astype(np.int32) if n else np.zeros(0, np.int32)
    n = len(keys)
    b = rng.permutation(n).astype(np.int64) if unique_b else rng.integers(0, 60, n)
    cols = [keys, b, _floats(rng, n), rng.integers(0, 6, n).astype(np.uint8), np.full(n, 1 << 40, dtype=np.int64)]
    return HostRelation("i", IN_NAMES, [P.INT4, P.INT8, P.FLOAT8, P.DICT8, P.INT8], cols,
                        nulls=[_nulls(rng, n, key_null), _nulls(rng, n, 0.1 if not unique_b else 0.0), None, None, None],
                        dict_texts=[None, None, None, TEXTS, None])


def make(fn, *a, **k):
    from oracle import oracle as O
    return fn(*a, **k).set_dict_hashes(O.hashbpchar), fn(*a, **k).set_dict_hashes(capi.hashbpchar)


def scan(relid, rel, names):
    return P.SeqScan(relid, [(nme, P.Var(relid, *rel.var(nme))) for nme in names])


def o(name):
    return P.OuterVar(OUT_NAMES.index(name) + 1, *{"k": (P.INT4,), "a": (P.INT8,), "f": (P.FLOAT8,), "s": (P.DICT8,), "e": (P.INT8,)}[name])


def i(name):
    return P.InnerVar(IN_NAMES.index(name) + 1, *{"ik": (P.INT4,), "b": (P.INT8,), "g": (P.FLOAT8,), "t": (P.DICT8,), "big": (P.INT8,)}[name])


FILTERS = {
    "ne": lambda: [P.OpExpr(P.OP_NE, o("a"), i("b"))],
    "lt": lambda: [P.OpExpr(P.OP_LT, o("a"), i("b"))],
    "eq": lambda: [P.OpExpr(P.OP_EQ, o("a"), i("b"))],
    "arith": lambda: [P.OpExpr(P.OP_LT, P.OpExpr(P.OP_ADD, o("a"), P.Const(P.INT8, 3)), i("b"))],
    "float_nan": lambda: [P.OpExpr(P.OP_LT, o("f"), i("g"))],
    "dict": lambda: [P.OpExpr(P.OP_EQ, o("s"), i("t"))],
    "or_not": lambda: [P.BoolExpr(P.OR_EXPR, P.OpExpr(P.OP_LT, o("a"), i("b")),
                                  P.BoolExpr(P.NOT_EXPR, P.OpExpr(P.OP_EQ, o("s"), i("t"))))],
    "one_side_each": lambda: [P.OpExpr(P.OP_GT, o("a"), P.Const(P.INT8, 20)), P.OpExpr(P.OP_LT, i("b"), P.Const(P.INT8, 40))],
}


def join_plan(jointype, fo, do, joinquals=(), quals=()):
    so = scan(1, fo, OUT_NAMES)
    si = scan(2, do, IN_NAMES)
    h = P.Hash(si, [P.out_var(si, 1)])
    targets = [(nme, o(nme)) for nme in OUT_NAMES[:4]]
    if jointype not in (P.JOIN_SEMI, P.JOIN_ANTI, P.JOIN_LASJ_NOTIN):
        targets += [(nme, i(nme)) for nme in IN_NAMES[:4]]
    return P.HashJoin(jointype, so, h, [P.out_var(so, 1)], targets, joinquals=list(joinquals), quals=list(quals))


def run(ctx, oracle, plan, rels_o, rels_p, generic, mem_kb=0):
    """(rows, kernel names launched, batch passes, largest nbatch) of the executor, and the oracle's rows"""
    dev = to_device(ctx, rels_p)
    ctx.check(ctx.L.cbgpu_rel_share_dict_hash(dev[1].h, IN_NAMES.index("t"), dev[0].h, OUT_NAMES.index("s")))
    ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
    ctx.trace_begin()
    try:
        got = ex.run(plan)
    finally:
        names = {nme for nme, _ in ctx.trace_end()}
        passes = int(ex.estate.contents.es_hashjoin_batches_run)
        ex.close()
        for d in dev:
            d.free()
    nb = max([v["hashjoin_nbatch"] for v in got.instrument.values()] + [1])
    return got.rows, names, passes, nb, oracle.execute(plan, [rels_o]).rows


def same(got, want):
    """exact, except that float8 NaN compares equal to itself"""
    key = lambda r: tuple("NaN" if isinstance(v, float) and math.isnan(v) else v for v in r)  # noqa: E731
    return canon([key(r) for r in got]) == canon([key(r) for r in want])


JOINS = [P.JOIN_LEFT, P.JOIN_SEMI, P.JOIN_ANTI]


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", JOINS)
@pytest.mark.parametrize("filt", sorted(FILTERS))
def test_filter_kinds(ctx, oracle, filt, jointype, generic):
    """every kind of filter, NULL keys and NULL filter inputs on both sides, three build rows per key"""
    fo, fp = make(outer_rel, 5003, 11, 400)
    do, dp = make(inner_rel, 1200, 12, 400, 3)
    plan = join_plan(jointype, fo, do, FILTERS[filt]())
    got, names, _, _, want = run(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert same(got, want)
    assert "k_ht_probe_filtered<count>" in names
    assert len(want) > 0


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", JOINS)
@pytest.mark.parametrize("dup", [1, 3, "skew"])
def test_duplicates_and_one_passing_candidate(ctx, oracle, dup, jointype, generic):
    """1 and 3 build rows per key, and every build row under one key with distinct b: `o.a = i.b` then lets exactly one of
    hundreds of candidates pass, wherever it lies in the chain"""
    fo, fp = make(outer_rel, 4001, 21, 8 if dup == "skew" else 400)
    do, dp = make(inner_rel, 600, 22, 400, dup, unique_b=dup == "skew")
    plan = join_plan(jointype, fo, do, FILTERS["eq"]())
    got, names, _, _, want = run(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert same(got, want) and "k_ht_probe_filtered<count>" in names
    if dup == "skew" and jointype == P.JOIN_SEMI:
        assert len(want) > 100


@pytest.mark.parametrize("nbatch", [1, 16])
@pytest.mark.parametrize("jointype", JOINS)
def test_filtered_pair_probe_finds_the_candidate_at_every_chain_position(ctx, oracle, jointype, nbatch):
    """all 600 build rows share one key and have distinct b; probe row r has a = r, so `o.a = i.b` lets exactly one candidate
    pass for each probe row, and over the 600 rows that candidate takes every position of the chain, the last one in slot order
    included.  SEMI must return each probe row with that one partner, ANTI none of them, LEFT one pair each."""
    L = ctx.L
    n = 600
    fo = HostRelation("o", OUT_NAMES, [P.INT4, P.INT8, P.FLOAT8, P.DICT8, P.INT8],
                      [np.full(n, 7, np.int32), np.arange(n), np.zeros(n), np.zeros(n, np.uint8), np.zeros(n, np.int64)],
                      dict_texts=[None, None, None, TEXTS, None]).set_dict_hashes(capi.hashbpchar)
    _, dp = make(inner_rel, n, 81, 10, "skew", unique_b=True, key_null=0.0)
    outer, inner = to_device(ctx, [fo, dp])
    keys = (C.c_int32 * 1)(0)
    filt = capi.join_filter([(outer, 1, 0), (inner, 1, 1)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_LOAD, 1, 0), (capi.CBP_EQ, 0, 0)])
    ht = C.c_void_p()
    ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, nbatch, C.byref(ht)))
    pairs, passes = capi.CbgpuPairs(), C.c_int64()
    ctx.check(L.cbgpu_ht_probe_pairs(ctx.h, ht, outer.h, keys, 1, jointype, C.byref(filt), None, None, C.byref(pairs),
                                     C.byref(passes)))
    a, b = _read_pairs(ctx, pairs)
    L.cbgpu_pairs_free(C.byref(pairs))
    L.cbgpu_ht_free(ht)
    outer.free()
    inner.free()
    if jointype == P.JOIN_ANTI:
        assert len(a) == 0
    else:
        partner = {int(v): r for r, v in enumerate(dp.columns[1].tolist())}      # build row whose b is v
        assert sorted(a.tolist()) == list(range(n)) and all(partner[int(r)] == int(c) for r, c in zip(a, b))


@pytest.mark.parametrize("jointype", JOINS)
@pytest.mark.parametrize("nf,nd", [(0, 500), (3000, 0), (0, 0)])
def test_empty_sides(ctx, oracle, jointype, nf, nd):
    fo, fp = make(outer_rel, nf, 31, 300)
    do, dp = make(inner_rel, nd, 32, 300, 3)
    plan = join_plan(jointype, fo, do, FILTERS["ne"]())
    got, _, _, _, want = run(ctx, oracle, plan, [fo, do], [fp, dp], False)
    assert same(got, want)
    assert len(want) == (nf if jointype != P.JOIN_SEMI else 0)


QUALS = {
    P.JOIN_INNER: lambda: [P.OpExpr(P.OP_LT, i("b"), P.Const(P.INT8, 40))],
    P.JOIN_LEFT: lambda: [P.OpExpr(P.OP_LT, i("b"), P.Const(P.INT8, 40))],
    P.JOIN_RIGHT: lambda: [P.OpExpr(P.OP_LT, o("a"), P.Const(P.INT8, 40))],
    P.JOIN_FULL: lambda: [P.OpExpr(P.OP_NE, o("a"), i("b"))],
    P.JOIN_SEMI: lambda: [P.OpExpr(P.OP_GT, o("a"), P.Const(P.INT8, 10))],
    P.JOIN_ANTI: lambda: [P.OpExpr(P.OP_GT, o("a"), P.Const(P.INT8, 10))],
    P.JOIN_LASJ_NOTIN: lambda: [P.OpExpr(P.OP_GT, o("a"), P.Const(P.INT8, 10))],
}


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype,with_filter", [(jt, wf) for jt in sorted(QUALS) for wf in (False, True)
                                                  if not (wf and jt not in JOINS)])
def test_plan_qual_on_non_inner_joins(ctx, oracle, jointype, with_filter, generic):
    """the plan's own qual filters joined and NULL-extended rows alike (a NULL inner value drops the row); with a join filter
    too where the join type takes one"""
    fo, fp = make(outer_rel, 4001, 41, 300)
    notin = jointype == P.JOIN_LASJ_NOTIN        # keys missing from the set, and no NULL in it (which would leave no row)
    do, dp = make(inner_rel, 900, 42, 600 if notin else 300, 3, key_null=0.0 if notin else 0.1)
    plan = join_plan(jointype, fo, do, FILTERS["lt"]() if with_filter else (), QUALS[jointype]())
    got, names, _, _, want = run(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert same(got, want) and len(want) > 0
    assert ("k_ht_probe_filtered<count>" in names) == with_filter


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", JOINS)
@pytest.mark.parametrize("dup", [1, 3])
def test_in_batches(ctx, oracle, jointype, dup, generic):
    """a 16 KB operator budget splits the build side: each probe row is decided in its own batch's pass, the same rows as
    without a budget and as the oracle"""
    fo, fp = make(outer_rel, 20011, 51, 3000)
    do, dp = make(inner_rel, 4000, 52, 3000, dup)
    plan = join_plan(jointype, fo, do, FILTERS["or_not"](), QUALS[jointype]())
    got, names, passes, nb, want = run(ctx, oracle, plan, [fo, do], [fp, dp], generic, mem_kb=16)
    free, _, _, nb1, _ = run(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert nb >= 4 and passes >= nb and nb1 == 1
    assert same(got, want) and same(free, want)
    assert "k_ht_probe_filtered<count>" in names


def test_overflow_in_the_filter(ctx, oracle):
    """o.e * i.big = 2^80 on every candidate: bigint out of range, not a wrapped product"""
    fo, fp = make(outer_rel, 2000, 61, 100)
    do, dp = make(inner_rel, 300, 62, 100, 3)
    plan = join_plan(P.JOIN_SEMI, fo, do, [P.OpExpr(P.OP_GT, P.OpExpr(P.OP_MUL, o("e"), i("big")), P.Const(P.INT8, 0))])
    with pytest.raises(capi.CbgpuError) as ei:
        run(ctx, oracle, plan, [fo, do], [fp, dp], False)
    assert ei.value.code == OVERFLOW


def _read_pairs(ctx, pairs):
    n = int(pairs.npairs)
    a = np.zeros(n, dtype=np.uint32)
    b = np.zeros(n, dtype=np.uint32)
    if n:
        ctx.check(ctx.L.cbgpu_read_u32(ctx.h, pairs.outer_idx, n, a.ctypes.data))
        ctx.check(ctx.L.cbgpu_read_u32(ctx.h, pairs.inner_idx, n, b.ctypes.data))
    return a.astype(np.int64), b.astype(np.int64)


def _brute(fo, do, jointype):
    """numpy nested loop: the filter `o.a <> i.b` over key-equal candidates, NULL keys and NULL a / b never pass"""
    ok, on, oa, oan = fo.columns[0], fo.nulls[0], fo.columns[1], fo.nulls[1]
    ik, inn, ib, ibn = do.columns[0], do.nulls[0], do.columns[1], do.nulls[1]
    passing = {}
    for r in range(len(ok)):
        if on[r]:
            continue
        cand = np.nonzero((ik == ok[r]) & (inn == 0))[0]
        ps = cand[(ibn[cand] == 0) & (oan[r] == 0) & (ib[cand] != oa[r])]
        if len(ps):
            passing[r] = set(ps.tolist())
    n = len(ok)
    if jointype == P.JOIN_SEMI:
        return passing
    if jointype == P.JOIN_ANTI:
        return {r for r in range(n) if r not in passing}
    return {(r, c) for r, s in passing.items() for c in s} | {(r, 0xFFFFFFFF) for r in range(n) if r not in passing}


@pytest.mark.parametrize("jointype", JOINS)
def test_pair_probe_against_a_nested_loop(ctx, jointype):
    """cbgpu_ht_probe_pairs: pairs in outer-row order, at most one per row for SEMI / ANTI, the same pairs from a
    one-batch table and from the same build side split into 16 batches, and the pairs a nested loop gives"""
    L = ctx.L
    fo, fp = make(outer_rel, 6007, 71, 500)
    do, dp = make(inner_rel, 1500, 72, 500, 3)
    outer, inner = to_device(ctx, [fp, dp])
    keys = (C.c_int32 * 1)(0)
    filt = capi.join_filter([(outer, 1, 0), (inner, 1, 1)], [(capi.CBP_LOAD, 0, 0), (capi.CBP_LOAD, 1, 0), (capi.CBP_NE, 0, 0)])
    want = _brute(fo, do, jointype)
    results = []
    for nbatch in (1, 16):
        ht = C.c_void_p()
        ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, nbatch, C.byref(ht)))
        pairs, passes = capi.CbgpuPairs(), C.c_int64()
        ctx.check(L.cbgpu_ht_probe_pairs(ctx.h, ht, outer.h, keys, 1, jointype, C.byref(filt), None, None, C.byref(pairs),
                                         C.byref(passes)))
        a, b = _read_pairs(ctx, pairs)
        L.cbgpu_pairs_free(C.byref(pairs))
        L.cbgpu_ht_free(ht)
        assert passes.value == (0 if nbatch == 1 else 16)
        runs = int((np.diff(a) < 0).sum()) + 1 if len(a) else 0
        assert runs <= nbatch                                     # ascending probe rows within each batch's pass
        if jointype != P.JOIN_LEFT:
            assert len(set(a.tolist())) == len(a)                 # at most one pair per probe row
        results.append(sorted(zip(a.tolist(), b.tolist())))
        if jointype == P.JOIN_SEMI:
            assert set(a.tolist()) == set(want) and all(int(c) in want[int(r)] for r, c in zip(a, b))
        elif jointype == P.JOIN_ANTI:
            assert set(a.tolist()) == want and set(b.tolist()) <= {0xFFFFFFFF}
        else:
            assert set(zip(a.tolist(), b.tolist())) == want and len(a) == len(want)
    if jointype != P.JOIN_SEMI:
        assert results[0] == results[1]
    else:
        assert [r for r, _ in results[0]] == [r for r, _ in results[1]]   # the first passing partner depends on slot order
    outer.free()
    inner.free()
