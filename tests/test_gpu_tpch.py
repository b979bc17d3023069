"""GPU parity tests proper (-m gpu): the CUDA path, through the C ABI and the ExecProcNode-style
executor, against (a) the reference's own expected rows for Q1/Q3/Q5 (tests/golden) and (b) the CPU
oracle on seeded synthetic tables.  Bit-exact: counts, keys, decimal sums and the numeric text."""
import numpy as np
import pytest

from cloudberry_b200 import capi, tpch
from cloudberry_b200 import plan as P
from gpu_util import canon, shard, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden_dev(ctx, golden):
    rels, exp = golden
    for r in rels:
        r.set_dict_hashes(capi.hashbpchar)      # product-side hashing of dictionary texts
    return to_device(ctx, rels), rels, exp


@pytest.mark.parametrize("generic", [False, True])
def test_q1_reference_expected(ctx, golden_dev, generic):
    dev, rels, exp = golden_dev
    ex = capi.Executor(ctx, dev, force_generic=generic)
    res = ex.run(tpch.q1_plan(1))
    assert tpch.format_q1(res.rows) == exp["q1"]
    kernels = sum(v["kernels"] for v in res.instrument.values())
    assert kernels > 0
    name, ms = ctx.last_kernel()
    ex.close()


@pytest.mark.parametrize("generic", [False, True])
def test_q3_reference_expected(ctx, golden_dev, generic):
    dev, rels, exp = golden_dev
    seg = exp["dict"]["c_mktsegment_dict"].index("MACHINERY")
    ex = capi.Executor(ctx, dev, force_generic=generic)
    res = ex.run(tpch.q3_plan(seg, 1))
    assert tpch.format_q3(res.rows) == exp["q3"]
    ex.close()


@pytest.mark.parametrize("generic", [False, True])
def test_q5_reference_expected(ctx, golden_dev, generic):
    dev, rels, exp = golden_dev
    reg = exp["dict"]["r_name_dict"].index("AMERICA")
    ex = capi.Executor(ctx, dev, force_generic=generic)
    res = ex.run(tpch.q5_plan(reg, 1))
    assert tpch.format_q5(res.rows, exp["dict"]["n_name_dict"]) == exp["q5"]
    ex.close()


@pytest.mark.parametrize("nsegs,generic", [pytest.param(n, g, id="%d%s" % (n, "-generic" if g else ""))
                                           for g in (False, True) for n in (2, 3)])
def test_q1_two_stage_on_segments(ctx, oracle, golden, nsegs, generic):
    """partial agg -> Redistribute Motion (cdbhash + jump hash on device) -> final agg -> gather, through the fused
    kernels' sinks and through the generic kernel's."""
    rels, exp = golden
    segs = shard(oracle, rels, nsegs)
    dsegs = [to_device(ctx, s) for s in segs]
    cl = capi.Cluster(ctx, dsegs, force_generic=generic)
    res = cl.run(tpch.q1_plan(nsegs))
    assert tpch.format_q1(res.rows) == exp["q1"]
    assert set(res.segments) == {0}
    cl.close()


@pytest.mark.parametrize("replicated,generic", [pytest.param(r, g, id="%s%s" % (r, "-generic" if g else ""))
                                               for g in (False, True) for r in (True, False)])
def test_q3_q5_on_segments(ctx, oracle, golden, replicated, generic):
    rels, exp = golden
    nsegs = 3
    dist = dict(tpch.DIST_KEY)
    if not replicated:
        dist["customer"] = "c_custkey"
        dist["supplier"] = "s_suppkey"
    segs = shard(oracle, rels, nsegs, dist)
    dsegs = [to_device(ctx, s) for s in segs]
    cl = capi.Cluster(ctx, dsegs, force_generic=generic)
    seg = exp["dict"]["c_mktsegment_dict"].index("MACHINERY")
    res = cl.run(tpch.q3_plan(seg, nsegs, customer_replicated=replicated))
    assert tpch.format_q3(res.rows) == exp["q3"]
    reg = exp["dict"]["r_name_dict"].index("AMERICA")
    res = cl.run(tpch.q5_plan(reg, nsegs, replicated=replicated))
    assert tpch.format_q5(res.rows, exp["dict"]["n_name_dict"]) == exp["q5"]
    cl.close()


def test_generator_matches_host(ctx):
    """device generator (csrc/gen.cu) == numpy generator (tpch.py), row for row."""
    sz = {"lineitem": 100003, "orders": 25013, "customer": 1501, "supplier": 101, "part": 2000}
    G = ctx.L
    li = capi.DeviceRelation(ctx, sz["lineitem"], [t for _, t in tpch.SCHEMA["lineitem"]])
    ctx.check(G.cbgpu_gen_lineitem(ctx.h, li.h, 42, 0, sz["supplier"], sz["part"]))
    host = tpch.gen_lineitem(42, sz["lineitem"], sz["supplier"], sz["part"])
    for i, (name, _) in enumerate(tpch.SCHEMA["lineitem"]):
        got, _ = li.read_column(i)
        assert np.array_equal(got, host[name]), name
    od = capi.DeviceRelation(ctx, sz["orders"], [t for _, t in tpch.SCHEMA["orders"]])
    ctx.check(G.cbgpu_gen_orders(ctx.h, od.h, 42, 0, sz["customer"]))
    host = tpch.gen_orders(42, sz["orders"], sz["customer"])
    for i, (name, _) in enumerate(tpch.SCHEMA["orders"]):
        got, _ = od.read_column(i)
        assert np.array_equal(got, host[name]), name
    cu = capi.DeviceRelation(ctx, sz["customer"], [t for _, t in tpch.SCHEMA["customer"]])
    ctx.check(G.cbgpu_gen_customer(ctx.h, cu.h, 42))
    host = tpch.gen_customer(42, sz["customer"])
    for i, (name, _) in enumerate(tpch.SCHEMA["customer"]):
        got, _ = cu.read_column(i)
        assert np.array_equal(got, host[name]), name
    for r in (li, od, cu):
        r.free()


@pytest.mark.parametrize("generic", [False, True])
def test_synthetic_vs_oracle(ctx, oracle, generic):
    """seeded synthetic SF0.02: CUDA path vs oracle, all three queries, exact."""
    rels_o = tpch.gen_tables(0.02, oracle.hashbpchar)
    rels_p = tpch.gen_tables(0.02, capi.hashbpchar)
    dev = to_device(ctx, rels_p)
    ex = capi.Executor(ctx, dev, force_generic=generic)
    for plan in (tpch.q1_plan(1), tpch.q3_plan(4, 1), tpch.q5_plan(1, 1)):
        want = oracle.execute(plan, [rels_o])
        got = ex.run(plan)
        if plan.plan.type == P.T_LimitSort:
            assert got.rows == want.rows
        else:
            assert canon(got.rows) == canon(want.rows)
    ex.close()
    for d in dev:
        d.free()


def test_exec_proc_node_batch(ctx, oracle, golden):
    """cb_ExecProcNodeBatch: a sub-tree's output as one device-resident column batch (here the lower join of
    Q3: orders (date qual) x customer (segment qual)), equal to the oracle's rows for the same plan node."""
    rels, exp = golden
    dev = to_device(ctx, rels)
    ex = capi.Executor(ctx, dev)
    seg = exp["dict"]["c_mktsegment_dict"].index("MACHINERY")
    cutoff = tpch.date_to_days(1995, 3, 15)
    cust = tpch._scan("customer", ["c_custkey"], [P.OpExpr(P.OP_EQ, tpch._svar("customer", "c_mktsegment"), P.Const(P.DICT8, seg))])
    orders = tpch._scan("orders", ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"],
                        [P.OpExpr(P.OP_LT, tpch._svar("orders", "o_orderdate"), P.Const(P.DATE, cutoff))])
    hc = P.Hash(cust, [P.out_var(cust, 1)])
    j1 = P.HashJoin(P.JOIN_INNER, orders, hc, [P.out_var(orders, 2)],
                    [("o_orderkey", P.out_var(orders, 1)), ("o_orderdate", P.out_var(orders, 3)),
                     ("o_shippriority", P.out_var(orders, 4))])
    batch = ex.run_batch(j1)
    want = oracle.execute(j1, [rels])
    assert batch.rows() == len(want.rows) > 0
    got = list(zip(*[batch.read_column(c)[0].tolist() for c in range(3)]))
    assert sorted(got) == sorted(tuple(r) for r in want.rows)
    # and a filtered scan with no join at all
    b2 = ex.run_batch(orders)
    w2 = oracle.execute(orders, [rels])
    assert sorted(zip(*[b2.read_column(c)[0].tolist() for c in range(4)])) == sorted(tuple(r) for r in w2.rows)
    batch.free()
    b2.free()
    ex.close()
    for d in dev:
        d.free()
