"""GROUP BY over five to eight columns on the GPU (-m gpu).

A join -> aggregate pipeline over 5, 6, 7 and 8 group keys of every key type (int4, int8, date, character(1), dict8, dict32,
numeric, float8 with -0 / NaN, NULLs) against a Python group-by of the same rows: through the compiled probe chain
(k_probe_chain) where its keys allow, through the interpreter (k_pipeline_generic), and under a 16 KB operator budget, where
the aggregation runs in partitions.  One or two keys, a numeric one among them, over a plain scan.  Nine keys are refused before any launch.  TPC-H Q10 (seven keys) and Q18 (five keys, its IN
subquery an aggregate with HAVING under a Hash) against the numpy answers of tpch_q10_q18 at SF0.01 on both routes and at
16 KB, at SF1 at their own LIMITs, and Q18 on a 3-segment cluster.  The CPU oracle does not hash numeric keys, and both
queries group by one, so numpy is their reference."""
import pytest

import wide_groups as W
from cloudberry_b200 import capi, tpch_q10_q18 as Q
from gpu_util import shard, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def run(ctx, rels, plan, generic=False, mem_kb=0):
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
    ctx.trace_begin()
    try:
        res = ex.run(plan)
    finally:
        names = [n for n, _ in ctx.trace_end()]
        ex.close()
        for d in dev:
            d.free()
    return res, names


def agg_kernel(names):
    """the kernel that filled the last aggregate table: the launch after its k_agg_init"""
    i = len(names) - 1 - names[::-1].index("k_agg_init")
    return names[i + 1]


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("nkeys", [5, 6, 7, 8])
def test_wide_groups_through_the_probe_chain(ctx, nkeys, mem_kb):
    rels = W.tables(20000, capi.hashbpchar)
    keys = W.CHAIN_KEYS[:nkeys]
    res, names = run(ctx, rels, W.plan(keys), mem_kb=mem_kb)
    assert W.canon(res.rows) == W.numpy_groups(rels[0], keys)
    if mem_kb and nkeys > 5:
        # the interpreter runs every partition's pass (five keys make 162 groups, which fit a 16 KB table)
        assert max(v["agg_npartitions"] for v in res.instrument.values()) > 1
        assert "k_pipeline_generic" in names
    else:
        assert "k_probe_chain" in names and "k_pipeline_generic" not in names


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("nkeys", [5, 6, 7, 8])
def test_wide_groups_with_nulls_and_float8_through_the_interpreter(ctx, nkeys, mem_kb):
    rels = W.tables(20000, capi.hashbpchar, nulls=True)
    keys = W.KEYS[:nkeys - 1] + ["k_f8"] if nkeys < 8 else W.KEYS[:8]
    res, names = run(ctx, rels, W.plan(keys), generic=True, mem_kb=mem_kb)
    assert W.canon(res.rows) == W.numpy_groups(rels[0], keys)
    assert "k_pipeline_generic" in names and "k_probe_chain" not in names
    assert (max(v["agg_npartitions"] for v in res.instrument.values()) > 1) == (mem_kb > 0)


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("keys", [["k_num"], ["k_num", "k_int4"]], ids=["num", "num_int4"])
def test_numeric_group_keys_over_a_scan(ctx, keys, generic):
    """one or two keys, a numeric one among them, with NULLs: the numeric key prints at its column's scale"""
    rels = W.tables(20000, capi.hashbpchar, nulls=True)
    res, names = run(ctx, rels, W.scan_plan(keys), generic=generic)
    assert W.canon(res.rows) == W.numpy_groups(rels[0], keys)
    assert {r[0] for r in res.rows} == {None, "-123.45", "0.00", "123.45"}
    if generic:
        assert agg_kernel(names) == "k_pipeline_generic"


def test_nine_keys_are_refused_before_any_launch(ctx):
    rels = W.tables(1000, capi.hashbpchar)
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev)
    before = ctx.launches()
    with pytest.raises(capi.CbgpuError) as e:
        ex.run(W.plan(W.KEYS))
    assert e.value.code == -3                      # CBGPU_ERR_UNSUPPORTED
    assert "GROUP BY with 9 columns is beyond the GPU path's limit (8)" in str(e.value)
    assert ctx.launches() == before
    ex.close()
    for d in dev:
        d.free()


Q18_SMALL = 250             # SF0.01 has few orders above 300 (an order has at most 7 lines of at most 50)


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("generic", [False, True])
def test_q10_q18_sf001_against_numpy(ctx, generic, mem_kb):
    rels = Q.gen_tables(0.01, capi.hashbpchar)
    # under the budget, whether a join runs in batches (the interpreter) depends on its build side's size: the kernel is pinned
    # without a budget only
    kernel = "k_pipeline_generic" if generic else "k_probe_chain"
    res, names = run(ctx, rels, Q.q10_plan(sf=0.01), generic, mem_kb)
    want = Q.q10_numpy_answer(0.01)
    assert [tuple(r) for r in res.rows] == want and len(want) == 20
    if not mem_kb:
        assert agg_kernel(names) == kernel
        assert names.count("k_agg_init") == 1          # the estimate held: one table, no retry after an overflow
    res, names = run(ctx, rels, Q.q18_plan(threshold=Q18_SMALL, sf=0.01), generic, mem_kb)
    want = Q.q18_numpy_answer(0.01, threshold=Q18_SMALL)
    assert [tuple(r) for r in res.rows] == want and len(want) >= 5
    if not mem_kb:
        assert agg_kernel(names) == kernel
        assert names.count("k_agg_init") == 2          # the subquery's table and the outer one


def test_q10_q18_sf1_against_numpy(ctx):
    rels = Q.gen_tables(1, capi.hashbpchar)
    res, names = run(ctx, rels, Q.q10_plan(sf=1))
    assert [tuple(r) for r in res.rows] == Q.q10_numpy_answer(1)
    assert agg_kernel(names) == "k_probe_chain" and names.count("k_agg_init") == 1
    res, names = run(ctx, rels, Q.q18_plan(sf=1))
    want = Q.q18_numpy_answer(1)
    assert [tuple(r) for r in res.rows] == want and len(want) >= 1
    assert agg_kernel(names) == "k_probe_chain" and names.count("k_agg_init") == 2
    assert sum(v["having_ms"] for v in res.instrument.values()) > 0      # the subquery's HAVING ran on the host, timed


def test_q18_on_three_segments(ctx, oracle):
    rels = Q.gen_tables(0.01, capi.hashbpchar)
    segs = shard(oracle, rels, 3, Q.DIST_KEY)
    devs = [to_device(ctx, s) for s in segs]
    cl = capi.Cluster(ctx, devs)
    try:
        got = [tuple(r) for r in cl.run(Q.q18_plan(threshold=Q18_SMALL, nsegs=3, sf=0.01)).rows]
    finally:
        cl.close()
        for d in devs:
            for r in d:
                r.free()
    assert got == Q.q18_numpy_answer(0.01, threshold=Q18_SMALL)
