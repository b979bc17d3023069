"""Pair-driven hash joins whose build side is split into batches (-m gpu): N:M INNER / LEFT joins and every RIGHT / FULL
join under an operator memory budget.  The probe side is partitioned by batch once, each batch is loaded and probed by its
own rows, and RIGHT / FULL keep one matched-row map across the passes (ExecHashJoinImpl's HJ_NEED_NEW_BATCH loop,
nodeHashjoin.c:709-738).  Every query is checked against the CPU oracle, which has no budget, and against the same executor
without a budget, through both kernel routes."""
import ctypes as C

import numpy as np
import pytest

from cloudberry_b200 import capi, tpch
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import canon, to_device
from test_gpu_edge import agg_over, dim, fact, make, scan

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def run_budgeted(ctx, oracle, plan, rels_o, rels_p, generic, mem_kb=16, split=True):
    """(rows under the budget, rows without one, the oracle's rows); asserts the build side was split when `split`"""
    dev = to_device(ctx, rels_p)
    ex = capi.Executor(ctx, dev, operator_mem_kb=mem_kb, force_generic=generic)
    ex1 = capi.Executor(ctx, dev, force_generic=generic)
    try:
        got = ex.run(plan)
        free = ex1.run(plan).rows
        batches = int(ex.estate.contents.es_hashjoin_batches_run)
    finally:
        ex.close()
        ex1.close()
        for d in dev:
            d.free()
    if split:
        nb = max(v["hashjoin_nbatch"] for v in got.instrument.values())
        assert nb >= 4 and batches > 0, (nb, batches)
    return got.rows, free, oracle.execute(plan, [rels_o]).rows


def _nm_join(jointype, fo, do):
    sf = scan(1, fo, ["k", "v", "amt", "g"])
    sd = scan(2, do, ["dk", "w", "c"])
    h = P.Hash(sd, [P.out_var(sd, 1)])
    return P.HashJoin(jointype, sf, h, [P.out_var(sf, 1)],
                      [("k", P.out_var(sf, 1)), ("g", P.out_var(sf, 4)), ("amt", P.out_var(sf, 3)), ("dk", P.InnerVar(1, P.INT4)),
                       ("w", P.InnerVar(2, P.INT8)), ("c", P.InnerVar(3, P.DICT8))])


NAMES = ["k", "g", "amt", "dk", "w", "c"]
AGGS = [("s", P.AGG_SUM, "amt"), ("n", P.AGG_COUNT_STAR, None), ("ck", P.AGG_COUNT, "k"), ("sw", P.AGG_SUM, "w")]


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", [P.JOIN_INNER, P.JOIN_LEFT])
def test_nm_inner_and_left_in_batches(ctx, oracle, jointype, generic):
    """duplicate build keys, NULL keys on both sides, 16 KB: every partner in its batch's pass, every NULL-extended LEFT row
    exactly once"""
    fo, fp = make(fact, 20011, seed=51, null_frac=0.1, kmax=3000)
    do, dp = make(dim, 4000, seed=52, null_frac=0.1, dup=3, kmax=3000)
    j = _nm_join(jointype, fo, do)
    got, free, want = run_budgeted(ctx, oracle, j, [fo, do], [fp, dp], generic)
    assert canon(got) == canon(want) == canon(free)
    assert len(want) > 20011 if jointype == P.JOIN_LEFT else len(want) > 0
    if jointype == P.JOIN_LEFT:
        assert any(r[0] is None and r[3] is None for r in want)        # NULL-keyed probe rows, NULL-extended
        assert any(r[0] is not None and r[3] is None for r in want)    # probe rows without a partner
    plan = agg_over(j, NAMES, ["g", "c"], AGGS)
    got, free, want = run_budgeted(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert canon(got) == canon(want) == canon(free)


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("dup", [1, 3])
@pytest.mark.parametrize("jointype", [P.JOIN_RIGHT, P.JOIN_FULL])
@pytest.mark.parametrize("nf,nd", [(0, 4000), (5000, 0), (3000, 4000), (20011, 9000), (400, 4500)])
def test_right_and_full_in_batches(ctx, oracle, jointype, nf, nd, dup, generic):
    """unmatched build rows (NULL-keyed ones included) come back once after all passes; FULL also keeps the unmatched probe
    rows, each in its own batch's pass"""
    kmax = nd // dup + 60
    fo, fp = make(fact, nf, seed=53, null_frac=0.1, kmax=kmax)
    do, dp = make(dim, nd, seed=54, null_frac=0.1, dup=dup, kmax=kmax)
    j = _nm_join(jointype, fo, do)
    got, free, want = run_budgeted(ctx, oracle, j, [fo, do], [fp, dp], generic, split=nd > 0)
    assert canon(got) == canon(want) == canon(free)
    if nd:
        assert any(r[0] is None and r[2] is None and r[3] is None for r in want)     # NULL-keyed build rows
    if nd and nf:
        assert any(r[0] is None and r[2] is None and r[3] is not None for r in want)  # unmatched build rows with a key
    if jointype == P.JOIN_FULL and nf:
        assert any(r[2] is not None and r[4] is None for r in want)                  # unmatched probe rows
    plan = agg_over(j, NAMES, ["g", "c"], AGGS)
    got, free, want = run_budgeted(ctx, oracle, plan, [fo, do], [fp, dp], generic, split=nd > 0)
    assert canon(got) == canon(want) == canon(free)


def _two_key_rel(name, n, seed, dup, null_frac):
    rng = np.random.default_rng(seed)
    if dup > 1:
        pairs = rng.permutation(50 * 100)[:n // dup]
        a, b = np.repeat(pairs // 100, dup)[:n], np.repeat(pairs % 100, dup)[:n]
    else:
        a, b = rng.integers(0, 50, n), rng.integers(0, 100, n)
    n = len(a)
    nulls = (rng.random(n) < null_frac).astype(np.uint8)
    return HostRelation(name, ["a", "b", "x"], [P.INT4, P.INT8, P.INT8], [a.astype(np.int32), b.astype(np.int64), rng.integers(0, 1000, n)],
                        nulls=[None, nulls, None])


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", [P.JOIN_INNER, P.JOIN_LEFT, P.JOIN_FULL])
def test_two_key_nm_join_in_batches(ctx, oracle, jointype, generic):
    """two join keys (int4, int8 with NULLs): the batch is the combined key hash's, on both sides alike"""
    fo, fp = make(_two_key_rel, "f2", 20011, 61, 1, 0.05)
    do, dp = make(_two_key_rel, "d2", 6000, 62, 3, 0.05)
    sf = scan(1, fo, ["a", "b", "x"])
    sd = scan(2, do, ["a", "b", "x"])
    h = P.Hash(sd, [P.out_var(sd, 1), P.out_var(sd, 2)])
    j = P.HashJoin(jointype, sf, h, [P.out_var(sf, 1), P.out_var(sf, 2)],
                   [("a", P.out_var(sf, 1)), ("b", P.out_var(sf, 2)), ("x", P.out_var(sf, 3)), ("ix", P.InnerVar(3, P.INT8))])
    got, free, want = run_budgeted(ctx, oracle, j, [fo, do], [fp, dp], generic)
    assert canon(got) == canon(want) == canon(free)
    assert len(want) > 20011 // 2


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("jointype", [P.JOIN_INNER, P.JOIN_LEFT, P.JOIN_FULL])
def test_one_key_holds_the_whole_build_side(ctx, oracle, jointype, generic):
    """skew: every build row has the same key, so one batch holds all of them and the other passes find nothing"""
    fo, fp = make(fact, 3000, seed=71, null_frac=0.1, kmax=50)
    do, dp = make(dim, 3000, seed=72, dup=3000, kmax=50)
    j = _nm_join(jointype, fo, do)
    plan = agg_over(j, NAMES, ["g", "c"], AGGS)
    got, free, want = run_budgeted(ctx, oracle, plan, [fo, do], [fp, dp], generic)
    assert canon(got) == canon(want) == canon(free)
    assert sum(int(r[3]) for r in want) > 3000 * 10


def _orders_lineitem(with_customer):
    so = tpch._scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"])
    sl = tpch._scan("lineitem", ["l_orderkey", "l_quantity", "l_extendedprice"])
    h = P.Hash(sl, [P.out_var(sl, 1)])
    j = P.HashJoin(P.JOIN_INNER, so, h, [P.out_var(so, 1)],
                   [("o_custkey", P.out_var(so, 2)), ("o_orderdate", P.out_var(so, 3)), ("l_quantity", P.InnerVar(2, *P.out_type(sl, 2))),
                    ("l_extendedprice", P.InnerVar(3, *P.out_type(sl, 3)))])
    names = ["o_custkey", "o_orderdate", "l_quantity", "l_extendedprice"]
    aggs = [("n", P.AGG_COUNT_STAR, None), ("sq", P.AGG_SUM, "l_quantity"), ("se", P.AGG_SUM, "l_extendedprice"),
            ("mx", P.AGG_MAX, "o_orderdate")]
    if not with_customer:
        v = tpch._child_var(j)
        return P.Agg(j, P.AGG_PLAIN, P.AGGSPLIT_SIMPLE, [], [(n, P.Aggref(op, None if a is None else v(a))) for n, op, a in aggs])
    sc = tpch._scan("customer", ["c_custkey", "c_mktsegment"])
    hc = P.Hash(sc, [P.out_var(sc, 1)])
    j2 = P.HashJoin(P.JOIN_INNER, j, hc, [P.out_var(j, 1)],
                    [(nme, P.out_var(j, i + 1)) for i, nme in enumerate(names)] + [("c_mktsegment", P.InnerVar(2, *P.out_type(sc, 2)))])
    return agg_over(j2, names + ["c_mktsegment"], ["c_mktsegment"], aggs)


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("mem_kb", [16, 1024])
def test_orders_join_lineitem_in_batches(ctx, oracle, mem_kb, generic):
    """SF0.05: orders probe Hash(lineitem) on l_orderkey (1-7 lines per order), aggregated; then the same pairs feed an N:1
    join to customer, itself split at 16 KB (its pipeline runs once per customer batch)"""
    rels_o = tpch.gen_tables(0.05, oracle.hashbpchar)
    rels_p = tpch.gen_tables(0.05, capi.hashbpchar)
    li, od = rels_o[0], rels_o[1]
    lines_with_order = int(np.isin(li.columns[li.attno("l_orderkey") - 1], od.columns[od.attno("o_orderkey") - 1]).sum())
    for with_customer in (False, True):
        plan = _orders_lineitem(with_customer)
        got, free, want = run_budgeted(ctx, oracle, plan, rels_o, rels_p, generic, mem_kb=mem_kb)
        assert canon(got) == canon(want) == canon(free)
        assert sum(int(r[-4]) for r in want) == lines_with_order      # each line once, with its order


def _read_pairs(ctx, pairs, ordered=False):
    n = int(pairs.npairs)
    o = np.zeros(n, dtype=np.uint32)
    i = np.zeros(n, dtype=np.uint32)
    if n:
        ctx.check(ctx.L.cbgpu_read_u32(ctx.h, pairs.outer_idx, n, o.ctypes.data))
        ctx.check(ctx.L.cbgpu_read_u32(ctx.h, pairs.inner_idx, n, i.ctypes.data))
    return (o, i) if ordered else sorted(zip(o.tolist(), i.tolist()))


def test_pair_order_is_deterministic(ctx):
    """the pair list comes out batch by batch, each batch's pairs in probe-row order, the unmatched build rows last: the same
    call twice gives the same probe-row sequence and the same pairs (the partners of one probe row come in the table's slot
    order, which each fill's concurrent inserts decide, as in the one-batch probe).  Rows of a query are a different matter:
    a MATERIALIZE sink appends in whatever order its warps finish, with or without batches."""
    L = ctx.L
    _, fp = make(fact, 20011, seed=81, null_frac=0.1, kmax=3000)
    _, dp = make(dim, 4000, seed=82, null_frac=0.1, dup=3, kmax=3000)
    outer, inner = to_device(ctx, [fp, dp])
    keys = (C.c_int32 * 1)(0)
    ht = C.c_void_p()
    ctx.check(L.cbgpu_ht_build_batched(ctx.h, inner.h, keys, 1, 32, C.byref(ht)))
    pairs, passes = capi.CbgpuPairs(), C.c_int64()
    for fill_outer, fill_inner in ((0, 0), (1, 1)):
        lists = []
        for _ in range(2):
            ctx.check(L.cbgpu_ht_probe_pairs_batched(ctx.h, ht, outer.h, keys, 1, fill_outer, fill_inner, None, None, C.byref(pairs),
                                                     C.byref(passes)))
            lists.append(_read_pairs(ctx, pairs, ordered=True))
            L.cbgpu_pairs_free(C.byref(pairs))
        (o, i), (o2, i2) = lists
        assert np.array_equal(o, o2) and sorted(zip(o.tolist(), i.tolist())) == sorted(zip(o2.tolist(), i2.tolist()))
        assert len(o) > 20011
        tail = o == 0xFFFFFFFF
        k = int(np.argmax(tail)) if tail.any() else len(o)
        assert (tail.any() and tail[k:].all()) if fill_inner else not tail.any()   # unmatched build rows behind all others
        assert (np.diff(o[:k].astype(np.int64)) < 0).sum() < 32          # at most one run of ascending probe rows per batch
    L.cbgpu_ht_free(ht)
    outer.free()
    inner.free()


def test_abi_batched_pair_probe(ctx):
    """cbgpu_ht_probe_pairs* refuse a multi-batch table (they would see one batch); cbgpu_ht_probe_pairs_batched over it
    returns the pair set a one-batch table over the same rows gives, for every fill_outer / fill_inner flavour"""
    L = ctx.L
    _, fp = make(fact, 20011, seed=91, null_frac=0.1, kmax=3000)
    _, dp = make(dim, 4000, seed=92, null_frac=0.1, dup=3, kmax=3000)
    outer, inner = to_device(ctx, [fp, dp])
    keys = (C.c_int32 * 1)(0)
    one, many = C.c_void_p(), C.c_void_p()
    ctx.check(L.cbgpu_ht_build(ctx.h, inner.h, keys, 1, C.byref(one)))
    ctx.check(L.cbgpu_ht_build_batched(ctx.h, inner.h, keys, 1, 16, C.byref(many)))
    assert L.cbgpu_ht_nbatch(one) == 1 and L.cbgpu_ht_nbatch(many) == 16
    pairs = capi.CbgpuPairs()
    rc = L.cbgpu_ht_probe_pairs(ctx.h, many, outer.h, keys, 1, None, 0, C.byref(pairs))
    assert rc == -2 and "cbgpu_ht_probe_pairs_batched" in ctx.error() and pairs.npairs == 0
    for fill_outer, fill_inner in ((0, 0), (1, 0), (0, 1), (1, 1)):
        rc = L.cbgpu_ht_probe_pairs_outer(ctx.h, many, outer.h, keys, 1, fill_outer, fill_inner, C.byref(pairs))
        assert rc == -2 and pairs.npairs == 0
        ctx.check(L.cbgpu_ht_probe_pairs_outer(ctx.h, one, outer.h, keys, 1, fill_outer, fill_inner, C.byref(pairs)))
        want = _read_pairs(ctx, pairs)
        L.cbgpu_pairs_free(C.byref(pairs))
        passes = C.c_int64()
        ctx.check(L.cbgpu_ht_probe_pairs_batched(ctx.h, many, outer.h, keys, 1, fill_outer, fill_inner, None, None, C.byref(pairs),
                                                 C.byref(passes)))
        got = _read_pairs(ctx, pairs)
        L.cbgpu_pairs_free(C.byref(pairs))
        assert passes.value == 16 and got == want and len(want) > 20011
    # the table stays usable as an N:1-style batched table: any batch can be made resident again
    ctx.check(L.cbgpu_ht_load_batch(many, 3))
    L.cbgpu_ht_free(one)
    L.cbgpu_ht_free(many)
    outer.free()
    inner.free()
