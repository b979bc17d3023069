"""Worker of tests/test_host_string_predicates_fake_runtime.py: LIKE / NOT LIKE / IN lists through libcbexec.so and libcbgpu.so
over the no-op runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host
memory).  Records each refusal's code, message and kernel launches, which kernels each accepted plan launches, and what a failing
device allocation leaves behind.  Prints one JSON object.  Not a test by itself."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from host_frees_worker import failing, plan_sweep, sweep  # noqa: E402

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402
from test_aocs_format import TCASES  # noqa: E402

VARCHAR = [b"", b"MEDIUM POLISHED TIN", b"PROMO BRUSHED", b"forest green", b"lime"]
BPCHAR = [b"SM BOX", b"SM CASE", b"ab"]
N = 1000


def main():
    out = {"refused": {}, "routes": {}, "calls": {}, "plans": {}}
    ctx = capi.Context(0)
    sweep.ctx = ctx
    sweep.msg = ""
    L = ctx.L
    dv = capi.DeviceDict.from_texts(ctx, VARCHAR)
    db = capi.DeviceDict.from_texts(ctx, BPCHAR, bpchar=True)

    def relation(dicts=True):
        rel = capi.DeviceRelation(ctx, N, [P.INT4, P.DICT32, P.DICT32, P.INT4])
        for c in range(4):
            col = np.ascontiguousarray(np.arange(N, dtype=np.int32) % [N, len(VARCHAR), len(BPCHAR), 50][c])
            L.cbgpu_rel_load_column(rel.h, c, col.ctypes.data, None)
        if dicts:
            rel.set_dict(1, dv, 0)
            rel.set_dict(2, db, 10)
        return rel

    rel, plain = relation(), relation(False)
    # a character(10) column decoded from a reference-written file: its dictionary is linked, its n is not declared
    ship = {c[0]: c for c in TCASES}["shipmode_bpchar10_nulls"]
    dship = capi.DeviceDict(ctx, max_entries=64)
    dship.collect(ship[5], ship[2])
    dship.finalize()
    decoded = capi.DeviceRelation(ctx, len(ship[6]), [P.INT4, P.DICT32])
    decoded.load_aocs_dict_column(1, ship[5], ship[2], dship)

    s, c, v = P.Var(1, 2, P.DICT32), P.Var(1, 3, P.DICT32), P.Var(1, 4, P.INT4)
    k = [P.Var(1, 1, P.INT4)]

    def refused(name, plan, rels):
        ex = capi.Executor(ctx, rels)
        before = ctx.launches()
        try:
            ex.run(plan)
            r = {"code": 0, "msg": ""}
        except capi.CbgpuError as e:
            r = {"code": e.code, "msg": str(e)}
        r["launches"] = ctx.launches() - before
        ex.close()
        out["refused"][name] = r

    def saop(var, op, use_or, vals):
        e = P.InList(var, vals)
        e.op, e.useOr = op, use_or
        return e

    for name, pred, rels in (
            ("malformed_pattern", P.Like(s, "ab\\"), [rel]),
            ("no_dictionary", P.Like(s, "ab%"), [plain]),
            ("not_a_string_column", P.Like(v, "ab%"), [rel]),
            ("bpchar_n_not_declared", P.Like(P.Var(1, 2, P.DICT32), "%AIR"), [decoded]),
            ("second_predicate_refused", P.BoolExpr(P.AND_EXPR, P.Like(s, "PROMO%"), P.Like(v, "x%")), [rel]),
            ("pattern_not_a_constant", P.Like(s, s), [rel]),
            ("array_op_lt", saop(v, P.OP_LT, True, [1, 2]), [rel]),
            ("array_eq_all", saop(v, P.OP_EQ, False, [1, 2]), [rel]),
            ("array_ne_any", saop(s, P.OP_NE, True, ["lime"]), [rel]),
            ("null_element", P.InList(v, [P.Const(P.INT4, 0, isnull=True), 1]), [rel]),
            ("null_string_element", P.InList(s, [P.Const(P.TEXT, 0, isnull=True), "lime"]), [rel]),
            ("mixed_elements", P.InList(s, ["lime", P.Const(P.DICT32, 1)]), [rel]),
            ("five_string_predicates", P.BoolExpr(P.OR_EXPR, *[P.Like(s, "%%%d" % i) for i in range(5)]), [rel])):
        refused(name, P.SeqScan(1, k, [pred]), rels)
    refused("text_constant_as_value", P.SeqScan(1, [P.TextConst("x")]), [rel])
    inner = P.SeqScan(2, [P.Var(2, 1, P.INT4), P.Var(2, 2, P.DICT32)])
    outer = P.SeqScan(1, k)
    h = P.Hash(inner, [P.out_var(inner, 1)])
    refused("above_a_join", P.HashJoin(P.JOIN_INNER, outer, h, [P.out_var(outer, 1)], [P.OuterVar(1, P.INT4)],
                                       quals=[P.Like(P.InnerVar(2, P.DICT32), "PROMO%")]), [rel, rel])

    # library calls refused before any launch
    def call(name, fn):
        before = ctx.launches()
        try:
            fn()
            r = {"code": 0, "msg": ""}
        except capi.CbgpuError as e:
            r = {"code": e.code, "msg": str(e)}
        r["launches"] = ctx.launches() - before
        out["refused"][name] = r

    call("texts_unsorted", lambda: capi.DeviceDict.from_texts(ctx, [b"b", b"a"]).free())
    call("texts_duplicate", lambda: capi.DeviceDict.from_texts(ctx, [b"a", b"a"]).free())
    call("texts_bpchar_trailing_blank", lambda: capi.DeviceDict.from_texts(ctx, [b"a "], bpchar=True).free())
    call("match_malformed_pattern", lambda: dv.match_like("a\\"))
    call("match_bpchar_without_n", lambda: db.match_like("SM%", 0))
    call("match_varchar_with_n", lambda: dv.match_like("SM%", 10))
    call("set_dict_bpchar_without_n", lambda: rel.set_dict(2, db, 0))
    call("match_ok", lambda: dv.match_like("%green%"))

    # accepted plans: which kernels they launch
    def route(name, plan, rels, generic=False, mem_kb=0):
        ex = capi.Executor(ctx, rels, force_generic=generic, operator_mem_kb=mem_kb)
        ctx.trace_begin()
        try:
            ex.run(plan)
            code = 0
        except capi.CbgpuError as e:
            code = e.code
        names = sorted({nme for nme, _ in ctx.trace_end()})
        ex.close()
        out["routes"][name] = {"code": code, "kernels": names}

    qual = P.BoolExpr(P.AND_EXPR, P.Like(s, "MEDIUM POLISHED%", negate=True), P.InList(c, ["SM CASE", "SM BOX  "]),
                      P.InList(v, [49, 14, 23, 45, 19, 3, 36, 9]))
    scan = P.SeqScan(1, [P.Var(1, 4, P.INT4)], [qual])
    agg = P.Agg(scan, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [P.OuterVar(1, P.INT4), P.Aggref(P.AGG_COUNT_STAR)], num_groups=64)
    for generic in (False, True):
        route("scan_agg" + ("_generic" if generic else ""), agg, [rel], generic)
    route("scan_agg_16kb", agg, [rel], mem_kb=16)
    build = P.SeqScan(2, [P.Var(2, 1, P.INT4)], [P.Like(P.Var(2, 2, P.DICT32), "%green%")])
    hb = P.Hash(build, [P.out_var(build, 1)])
    join = P.HashJoin(P.JOIN_INNER, outer, hb, [P.out_var(outer, 1)], [P.OuterVar(1, P.INT4)])
    route("build_side", join, [rel, rel])
    cl = capi.Cluster(ctx, [[rel], [rel], [rel]])
    ctx.trace_begin()
    try:
        cl.run(P.Motion(scan, P.MOTIONTYPE_GATHER))
        code = 0
    except capi.CbgpuError as e:
        code = e.code
    out["routes"]["cluster_3seg"] = {"code": code, "kernels": sorted({nme for nme, _ in ctx.trace_end()})}
    cl.close()

    # every device allocation failing in turn: NOMEM, nothing left behind, the next call succeeds
    def call_sweep(fn):
        def attempt(n):
            try:
                failing(n, fn)
                return 0, None
            except capi.CbgpuError as e:
                return e.code, None
        return sweep(attempt)

    out["calls"]["dict_from_texts"] = call_sweep(lambda: capi.DeviceDict.from_texts(ctx, VARCHAR).free())
    out["calls"]["dict_match_like"] = call_sweep(lambda: dv.match_like("%green%"))
    out["plans"]["scan_agg"] = plan_sweep(lambda: capi.Executor(ctx, [rel]), agg)
    out["plans"]["build_side"] = plan_sweep(lambda: capi.Executor(ctx, [rel, rel]), join)
    print("HOSTSTRINGS " + json.dumps(out))


if __name__ == "__main__":
    main()
