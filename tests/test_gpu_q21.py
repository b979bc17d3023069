"""TPC-H Q21 on the GPU (-m gpu): its Hash Semi Join and Hash Anti Join carry the join filter `l_suppkey <> l1.l_suppkey`, so
both run through the filtered pair probe (k_ht_probe_filtered).  SF0.01 against the CPU oracle through both kernel routes and
under a 16 KB operator budget; SF1 against tpch_q21.numpy_answer, rows in the query's order.  The device top-N takes LIMIT <= 64, so these runs
ask for the first 64 rows (tpch_q21.DEVICE_LIMIT) instead of 100."""
import pytest

from cloudberry_b200 import capi, tpch_q21
from gpu_util import to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def run_q21(ctx, sf, generic=False, mem_kb=0):
    dev = to_device(ctx, tpch_q21.gen_tables(sf, capi.hashbpchar))
    ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=mem_kb)
    ctx.trace_begin()
    try:
        res = ex.run(tpch_q21.q21_plan(limit=tpch_q21.DEVICE_LIMIT))
    finally:
        names = [n for n, _ in ctx.trace_end()]
        ex.close()
        for d in dev:
            d.free()
    nb = max(v["hashjoin_nbatch"] for v in res.instrument.values())
    return [tuple(r) for r in res.rows], names, nb


@pytest.mark.parametrize("mem_kb", [0, 16])
@pytest.mark.parametrize("generic", [False, True])
def test_q21_sf001_against_the_oracle(ctx, oracle, generic, mem_kb):
    want = [tuple(r) for r in oracle.execute(tpch_q21.q21_plan(limit=tpch_q21.DEVICE_LIMIT), [tpch_q21.gen_tables(0.01, oracle.hashbpchar)]).rows]
    got, names, nb = run_q21(ctx, 0.01, generic, mem_kb)
    assert got == want and len(want) >= 1
    assert names.count("k_ht_probe_filtered<count>") >= 2          # the semi join and the anti join
    assert (nb >= 4) == (mem_kb > 0)


def test_q21_sf1_against_numpy(ctx):
    got, names, _ = run_q21(ctx, 1)
    want = tpch_q21.numpy_answer(1, limit=tpch_q21.DEVICE_LIMIT)
    assert got == want and len(want) == tpch_q21.DEVICE_LIMIT
    assert "k_ht_probe_filtered<count>" in names
