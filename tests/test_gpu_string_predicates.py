"""LIKE, NOT LIKE and IN lists over dictionary-coded string columns on the GPU.

cbgpu_dict_match_like's bitmap (k_dict_like) is held against the regular-expression reference of tests/test_like_host.py over
dictionaries of 0 to 10^6 entries, entries longer than 1 KB, and character(n) and varchar dictionaries.  The executor's
translation (a code set per predicate, tested per row by INSET on the generic pipeline kernel) is held against a plain
Python row loop with SQL's three-valued logic, with the predicate in the qual of the driving scan and of a hash join's build
side, on both kernel routes, under a 16 KB operator budget, and on a 3-segment cluster."""
import random
import re

import numpy as np
import pytest

from cloudberry_b200 import capi
from cloudberry_b200 import plan as P
from test_like_host import ALPHABET, like_ref, make_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _dict_texts(rng, n, bpchar, maxlen=10, long_every=0):
    out = set()
    while len(out) < n:
        k = 1500 if long_every and len(out) % long_every == 0 else rng.randrange(0, maxlen)
        t = "".join(rng.choice(ALPHABET) for _ in range(k))
        if bpchar:
            t = t.rstrip(" ")
        out.add(t.encode())
    return sorted(out)


def like_matcher(pattern):
    """like_ref for one pattern over many texts without regex backtracking (which is cubic in a 1.5 KB text for '%a%a%a%'):
    the pattern splits at `%` into stretches of fixed character length, each a compiled regular expression; the first must
    match at the start, the last at the end, the ones between are found leftmost in turn.  None for a malformed pattern."""
    segs, cur, i = [], [], 0
    while i < len(pattern):
        ch = pattern[i]
        if ch == "\\":
            if i + 1 >= len(pattern):
                return None
            cur.append(re.escape(pattern[i + 1]))
            i += 2
            continue
        if ch == "%":
            segs.append(cur)
            cur = []
        else:
            cur.append("." if ch == "_" else re.escape(ch))
        i += 1
    segs.append(cur)
    rx = [re.compile("".join(s), re.DOTALL) for s in segs]
    lens = [len(s) for s in segs]

    def match(text, bpchar_len):
        s = text + " " * max(0, bpchar_len - len(text)) if bpchar_len else text
        if len(rx) == 1:
            return rx[0].fullmatch(s) is not None
        if sum(lens) > len(s) or not rx[0].match(s) or not rx[-1].fullmatch(s, len(s) - lens[-1]):
            return False
        pos, end = lens[0], len(s) - lens[-1]
        for r, n in zip(rx[1:-1], lens[1:-1]):
            m = r.search(s, pos, end)
            if not m:
                return False
            pos = m.start() + n
        return True
    return match


def _bitmap_cases(rng, texts, bpchar_len, patterns):
    d_texts = [t.decode() for t in texts]
    for pat in patterns:
        m = like_matcher(pat)
        yield pat, [None] * len(d_texts) if m is None else [m(t, bpchar_len) for t in d_texts]


def test_segment_reference_agrees_with_regex_reference():
    rng = random.Random(3)
    for text, bp, pat in make_cases(rng, 20000):
        m = like_matcher(pat)
        assert (None if m is None else m(text, bp)) == like_ref(text, bp, pat), (text, bp, pat)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1000, 10 ** 6])
@pytest.mark.parametrize("bpchar", [False, True])
def test_dict_like_bitmap(ctx, n, bpchar):
    rng = random.Random(n * 2 + bpchar)
    texts = _dict_texts(rng, n, bpchar, long_every=97 if n == 1000 else 0)
    bpchar_len = (max([len(t.decode()) for t in texts] + [0]) + 2) if bpchar else 0
    d = capi.DeviceDict.from_texts(ctx, texts, bpchar=bpchar)
    try:
        assert d.nentries() == n
        patterns = [p for _, _, p in make_cases(rng, 400 if n <= 1000 else 6)]
        patterns += ["%", "%a%", "_%", "a%", "%\\%%", "%" + " " * 2]
        for pat, want in _bitmap_cases(rng, texts, bpchar_len, patterns):
            if None in want or (n == 0 and like_ref("", 0, pat) is None):
                with pytest.raises(capi.CbgpuError) as ei:
                    d.match_like(pat, bpchar_len)
                assert ei.value.code == -2, str(ei.value)
                continue
            assert d.match_like(pat, bpchar_len) == want, pat
    finally:
        d.free()


# ---- the executor: one relation, string columns as codes ----
VARCHAR_TEXTS = sorted({t.encode() for t in ["", "PROMO BRUSHED TIN", "PROMO PLATED", "MEDIUM POLISHED STEEL", "forest green",
                                             "green", "lime", "SM CASE", "a%b", "a_b", "é€𝄞", "ab"]})
BPCHAR_TEXTS = sorted({t.encode() for t in ["SM CASE", "SM BOX", "SM PACK", "LG CASE", "MED BAG", "ab", "a", ""]})
BPCHAR_N = 10
NROWS = 20000


def _table(seed=5):
    rng = np.random.default_rng(seed)
    k = np.arange(NROWS, dtype=np.int32)
    s = rng.integers(0, len(VARCHAR_TEXTS), NROWS).astype(np.int32)
    c = rng.integers(0, len(BPCHAR_TEXTS), NROWS).astype(np.int32)
    v = rng.integers(0, 50, NROWS).astype(np.int32)
    s_null = (rng.random(NROWS) < 0.1).astype(np.uint8)
    c_null = (rng.random(NROWS) < 0.1).astype(np.uint8)
    return k, s, c, v, s_null, c_null


def _load(ctx, rows, dicts):
    k, s, c, v, s_null, c_null = rows
    rel = capi.DeviceRelation(ctx, len(k), [P.INT4, P.DICT32, P.DICT32, P.INT4])
    for i, (col, nl) in enumerate(((k, None), (s, s_null), (c, c_null), (v, None))):
        col = np.ascontiguousarray(col)
        nlp = np.ascontiguousarray(nl) if nl is not None else None
        ctx.check(ctx.L.cbgpu_rel_load_column(rel.h, i, col.ctypes.data, nlp.ctypes.data if nlp is not None else None))
    rel.set_dict(1, dicts[0], 0)
    rel.set_dict(2, dicts[1], BPCHAR_N)
    ctx.sync()
    return rel


# predicates as (plan builder over scanrelid, python evaluator over one row -> True / False / None)
def _s(r):
    return None if r["s_null"] else VARCHAR_TEXTS[r["s"]].decode()


def _c(r):
    return None if r["c_null"] else BPCHAR_TEXTS[r["c"]].decode()


def _like(val, n, pat, neg=False):
    if val is None:
        return None
    m = like_ref(val, n, pat)
    return (not m) if neg else m


def _in(val, lst, neg=False, pad=False):
    if val is None:
        return None
    norm = (lambda x: x.rstrip(" ")) if pad else (lambda x: x)
    m = any(norm(val) == norm(x) for x in lst)
    return (not m) if neg else m


def _and(*xs):
    if any(x is False for x in xs):
        return False
    return None if any(x is None for x in xs) else True


def _or(*xs):
    if any(x is True for x in xs):
        return True
    return None if any(x is None for x in xs) else False


def _not(x):
    return None if x is None else not x


def _preds(rid):
    s = P.Var(rid, 2, P.DICT32)
    c = P.Var(rid, 3, P.DICT32)
    v = P.Var(rid, 4, P.INT4)
    cont = ["SM CASE", "SM BOX  ", "SM PACK", "SM PKG"]
    return {
        "like_prefix": (P.Like(s, "PROMO%"), lambda r: _like(_s(r), 0, "PROMO%"), True),
        "like_infix": (P.Like(s, "%green%"), lambda r: _like(_s(r), 0, "%green%"), True),
        "notlike": (P.Like(s, "MEDIUM POLISHED%", negate=True), lambda r: _like(_s(r), 0, "MEDIUM POLISHED%", True), True),
        "like_escape": (P.Like(s, "a\\%b"), lambda r: _like(_s(r), 0, "a\\%b"), True),
        "like_utf8": (P.Like(s, "_€%"), lambda r: _like(_s(r), 0, "_€%"), True),
        "bpchar_like_exact": (P.Like(c, "ab"), lambda r: _like(_c(r), BPCHAR_N, "ab"), True),
        "bpchar_like_pad": (P.Like(c, "ab%"), lambda r: _like(_c(r), BPCHAR_N, "ab%"), True),
        "bpchar_like_blanks": (P.Like(c, "SM CASE   "), lambda r: _like(_c(r), BPCHAR_N, "SM CASE   "), True),
        "in_bpchar": (P.InList(c, cont), lambda r: _in(_c(r), cont, pad=True), False),
        "notin_varchar": (P.InList(s, ["lime", "green", "nowhere"], negate=True), lambda r: _in(_s(r), ["lime", "green", "nowhere"], True), False),
        "in_int": (P.InList(v, [49, 14, 23, 45, 19, 3, 36, 9]), lambda r: r["v"] in (49, 14, 23, 45, 19, 3, 36, 9), False),
        "notin_int": (P.InList(v, [1, 2, 3], negate=True), lambda r: r["v"] not in (1, 2, 3), False),
        "and_or_not": (P.BoolExpr(P.OR_EXPR, P.BoolExpr(P.AND_EXPR, P.InList(c, cont), P.Like(s, "PROMO%", negate=True)),
                                  P.BoolExpr(P.NOT_EXPR, P.Like(c, "%A%"))),
                       lambda r: _or(_and(_in(_c(r), cont, pad=True), _like(_s(r), 0, "PROMO%", True)), _not(_like(_c(r), BPCHAR_N, "%A%"))),
                       True),
    }


def _rows_dicts(rows):
    k, s, c, v, s_null, c_null = rows
    return [dict(k=int(k[i]), s=int(s[i]), c=int(c[i]), v=int(v[i]), s_null=bool(s_null[i]), c_null=bool(c_null[i]))
            for i in range(len(k))]


def _want(rows, fn):
    return sorted(r["k"] for r in _rows_dicts(rows) if fn(r) is True)


@pytest.fixture(scope="module")
def setup(ctx):
    rows = _table()
    dicts = [capi.DeviceDict.from_texts(ctx, VARCHAR_TEXTS), capi.DeviceDict.from_texts(ctx, BPCHAR_TEXTS, bpchar=True)]
    rel = _load(ctx, rows, dicts)
    probe = capi.DeviceRelation(ctx, NROWS, [P.INT4])
    pk = np.ascontiguousarray(np.random.default_rng(9).permutation(NROWS).astype(np.int32))
    ctx.check(ctx.L.cbgpu_rel_load_column(probe.h, 0, pk.ctypes.data, None))
    ctx.sync()
    yield rows, dicts, rel, probe
    rel.free()
    probe.free()
    for d in dicts:
        d.free()


def _run(ctx, ex, plan):
    ctx.trace_begin()
    try:
        got = ex.run(plan)
    finally:
        names = {nme for nme, _ in ctx.trace_end()}
    return sorted(int(r[0]) for r in got.rows), names


@pytest.mark.parametrize("generic,mem_kb", [(False, 0), (True, 0), (False, 16)])
@pytest.mark.parametrize("name", list(_preds(1)))
def test_scan_qual(ctx, setup, name, generic, mem_kb):
    rows, _, rel, _ = setup
    pred, fn, like = _preds(1)[name]
    plan = P.SeqScan(1, [P.Var(1, 1, P.INT4)], [pred])
    ex = capi.Executor(ctx, [rel], force_generic=generic, operator_mem_kb=mem_kb)
    try:
        got, names = _run(ctx, ex, plan)
    finally:
        ex.close()
    assert got == _want(rows, fn)
    assert "k_pipeline_generic" in names, names
    assert ("k_dict_like" in names) == like, names


@pytest.mark.parametrize("generic,mem_kb", [(False, 0), (True, 0), (False, 16)])
@pytest.mark.parametrize("name", ["like_infix", "notlike", "in_bpchar", "and_or_not"])
def test_build_side_qual(ctx, setup, name, generic, mem_kb):
    """the predicate filters the build side of a hash join; the probe side is a permutation of the keys"""
    rows, _, rel, probe = setup
    pred, fn, like = _preds(2)[name]
    outer = P.SeqScan(1, [P.Var(1, 1, P.INT4)])
    inner = P.SeqScan(2, [P.Var(2, 1, P.INT4)], [pred])
    h = P.Hash(inner, [P.out_var(inner, 1)])
    plan = P.HashJoin(P.JOIN_INNER, outer, h, [P.out_var(outer, 1)], [P.OuterVar(1, P.INT4)])
    ex = capi.Executor(ctx, [probe, rel], force_generic=generic, operator_mem_kb=mem_kb)
    try:
        got, names = _run(ctx, ex, plan)
    finally:
        ex.close()
    assert got == _want(rows, fn)
    assert "k_pipeline_generic" in names and ("k_dict_like" in names) == like, names


@pytest.mark.parametrize("name", ["like_prefix", "bpchar_like_pad", "in_bpchar", "and_or_not"])
def test_cluster_of_three(ctx, setup, name):
    """a table distributed over three segments: each segment's relation links the same dictionaries"""
    rows, dicts, _, _ = setup
    pred, fn, like = _preds(1)[name]
    segs = []
    for g in range(3):
        idx = np.nonzero(rows[0] % 3 == g)[0]
        segs.append(_load(ctx, tuple(np.ascontiguousarray(a[idx]) for a in rows), dicts))
    try:
        scan = P.SeqScan(1, [P.Var(1, 1, P.INT4)], [pred])
        plan = P.Motion(scan, P.MOTIONTYPE_GATHER)
        cl = capi.Cluster(ctx, [[r] for r in segs])
        ctx.trace_begin()
        try:
            got = cl.run(plan)
        finally:
            names = {nme for nme, _ in ctx.trace_end()}
            cl.close()
        assert sorted(int(r[0]) for r in got.rows) == _want(rows, fn)
        assert "k_pipeline_generic" in names and ("k_dict_like" in names) == like, names
    finally:
        for r in segs:
            r.free()


def test_refusals(ctx, setup):
    """before any launch: a malformed pattern, LIKE over a column without a dictionary or a non-string column, other
    array operators, NULL elements"""
    _, _, rel, _ = setup
    plain = capi.DeviceRelation(ctx, 4, [P.INT4, P.DICT32])
    cases = [
        (rel, P.Like(P.Var(1, 2, P.DICT32), "ab\\"), -2),
        (plain, P.Like(P.Var(1, 2, P.DICT32), "ab%"), -3),
        (rel, P.Like(P.Var(1, 4, P.INT4), "ab%"), -3),
        (rel, _saop(P.Var(1, 4, P.INT4), P.OP_LT, True, [1, 2]), -3),
        (rel, _saop(P.Var(1, 4, P.INT4), P.OP_EQ, False, [1, 2]), -3),
        (rel, P.InList(P.Var(1, 4, P.INT4), [P.Const(P.INT4, 0, isnull=True), P.Const(P.INT4, 1)]), -3),
    ]
    try:
        for r, pred, code in cases:
            ex = capi.Executor(ctx, [r])
            before = ctx.launches()
            try:
                with pytest.raises(capi.CbgpuError) as ei:
                    ex.run(P.SeqScan(1, [P.Var(1, 1, P.INT4)], [pred]))
                assert ei.value.code == code, str(ei.value)
                assert ctx.launches() == before
            finally:
                ex.close()
    finally:
        plain.free()


def _saop(var, op, use_or, vals):
    e = P.InList(var, vals)
    e.op = op
    e.useOr = use_or
    return e


def test_decoded_bpchar_column_needs_its_length(ctx):
    """a character(10) column decoded from a reference-written file: LIKE is refused until the loader declares n (matching the
    blank-trimmed dictionary entries unpadded would make 'REG AIR'::char(10) LIKE '%AIR' true); with n declared the rows
    are the padded reference's"""
    from test_aocs_format import TCASES
    ship = {c[0]: c for c in TCASES}["shipmode_bpchar10_nulls"]
    values, nulls = ship[6], ship[7]
    d = capi.DeviceDict(ctx, max_entries=64)
    d.collect(ship[5], ship[2])
    d.finalize()
    rel = capi.DeviceRelation(ctx, len(values), [P.INT4, P.DICT32])
    k = np.ascontiguousarray(np.arange(len(values), dtype=np.int32))
    ctx.check(ctx.L.cbgpu_rel_load_column(rel.h, 0, k.ctypes.data, None))
    rel.load_aocs_dict_column(1, ship[5], ship[2], d)
    try:
        for pat in ("%AIR", "%AIR%", "REG AIR", "REG AIR   ", "_AIL%"):
            plan = P.SeqScan(1, [P.Var(1, 1, P.INT4)], [P.Like(P.Var(1, 2, P.DICT32), pat)])
            ex = capi.Executor(ctx, [rel])
            try:
                before = ctx.launches()
                with pytest.raises(capi.CbgpuError) as ei:
                    ex.run(plan)
                assert ei.value.code == -3 and "not declared" in str(ei.value) and ctx.launches() == before
            finally:
                ex.close()
        rel.set_dict(1, d, 10)
        for pat in ("%AIR", "%AIR%", "REG AIR", "REG AIR   ", "_AIL%"):
            ex = capi.Executor(ctx, [rel])
            try:
                got = sorted(int(r[0]) for r in ex.run(P.SeqScan(1, [P.Var(1, 1, P.INT4)], [P.Like(P.Var(1, 2, P.DICT32), pat)])).rows)
            finally:
                ex.close()
            want = [i for i, (v, z) in enumerate(zip(values, nulls)) if not z and like_ref(v.rstrip(b" ").decode(), 10, pat)]
            assert got == want, pat
    finally:
        rel.free()
        d.free()
