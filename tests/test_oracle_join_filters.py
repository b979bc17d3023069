"""The oracle's hash joins with a join filter (joinqual) and with the plan's own qual (oracle/oracle.c hashjoin_next,
nodeHashjoin.c:583-713) against a brute-force nested loop in plain Python, and the oracle's TPC-H Q21 against an independent
numpy evaluation of the SQL: the check that the checker is right before the CUDA path is compared with it
(tests/test_gpu_join_filters.py, tests/test_gpu_q21.py).

SQL semantics restated here: a NULL join key never matches; a filter or qual that is NULL counts as false (ExecQual); float8
compares with every NaN equal and above everything (float8_cmp_internal); SEMI keeps a probe row with at least one passing
candidate, ANTI one with none, LEFT every passing pair or one NULL-extended row; RIGHT / FULL add the unmatched build rows;
NOT IN returns nothing when the set holds a NULL, drops a NULL probe key unless the set is empty."""
import math

import pytest

from cloudberry_b200 import plan as P
from cloudberry_b200 import tpch_q21
from test_gpu_join_filters import FILTERS, IN_NAMES, OUT_NAMES, QUALS, inner_rel, join_plan, outer_rel


def _cmp(x, y):
    if x is None or y is None:
        return None
    if isinstance(x, float) and math.isnan(x):
        return 0 if isinstance(y, float) and math.isnan(y) else 1
    if isinstance(y, float) and math.isnan(y):
        return -1
    return (x > y) - (x < y)


def _op(test):
    return lambda x, y: None if _cmp(x, y) is None else test(_cmp(x, y))


EQ, NE, LT, GT = _op(lambda c: c == 0), _op(lambda c: c != 0), _op(lambda c: c < 0), _op(lambda c: c > 0)


def AND(x, y):
    return False if x is False or y is False else (None if x is None or y is None else True)


def OR(x, y):
    return True if x is True or y is True else (None if x is None or y is None else False)


def NOT(x):
    return None if x is None else not x


def ADD(x, y):
    return None if x is None or y is None else x + y


PY_FILTERS = {
    "ne": lambda o, i: NE(o["a"], i["b"]),
    "lt": lambda o, i: LT(o["a"], i["b"]),
    "eq": lambda o, i: EQ(o["a"], i["b"]),
    "arith": lambda o, i: LT(ADD(o["a"], 3), i["b"]),
    "float_nan": lambda o, i: LT(o["f"], i["g"]),
    "dict": lambda o, i: EQ(o["s"], i["t"]),
    "or_not": lambda o, i: OR(LT(o["a"], i["b"]), NOT(EQ(o["s"], i["t"]))),
    "one_side_each": lambda o, i: AND(GT(o["a"], 20), LT(i["b"], 40)),
}
PY_QUALS = {
    P.JOIN_INNER: lambda o, i: LT(i["b"], 40),
    P.JOIN_LEFT: lambda o, i: LT(i["b"], 40),
    P.JOIN_RIGHT: lambda o, i: LT(o["a"], 40),
    P.JOIN_FULL: lambda o, i: NE(o["a"], i["b"]),
    P.JOIN_SEMI: lambda o, i: GT(o["a"], 10),
    P.JOIN_ANTI: lambda o, i: GT(o["a"], 10),
    P.JOIN_LASJ_NOTIN: lambda o, i: GT(o["a"], 10),
}


def _rows(rel, names):
    cols = []
    for c in range(len(names)):
        vals = rel.columns[c].tolist()
        nl = rel.nulls[c].tolist() if rel.nulls[c] is not None else [0] * len(vals)
        cols.append([None if n else v for v, n in zip(vals, nl)])
    return [dict(zip(names, r)) for r in zip(*cols)] if cols and cols[0] else []


def brute(jointype, fo, do, filt=None, qual=None):
    """the rows of join_plan(jointype, fo, do, filter, qual) by a nested loop"""
    orows, irows = _rows(fo, OUT_NAMES), _rows(do, IN_NAMES)
    nul_o, nul_i = dict.fromkeys(OUT_NAMES), dict.fromkeys(IN_NAMES)
    f = filt or (lambda o, i: True)
    q = qual or (lambda o, i: True)
    inner_out = jointype not in (P.JOIN_SEMI, P.JOIN_ANTI, P.JOIN_LASJ_NOTIN)

    def row(o, i):
        return tuple(o[n] for n in OUT_NAMES[:4]) + (tuple(i[n] for n in IN_NAMES[:4]) if inner_out else ())
    out = []
    if jointype == P.JOIN_LASJ_NOTIN:
        keys = [i["ik"] for i in irows]
        if None in keys:
            return []
        return [row(o, nul_i) for o in orows if (not keys or (o["k"] is not None and o["k"] not in keys)) and q(o, nul_i) is True]
    matched = set()
    for o in orows:
        hits = [j for j, i in enumerate(irows) if o["k"] is not None and o["k"] == i["ik"] and f(o, irows[j]) is True]
        matched.update(hits)
        if jointype == P.JOIN_SEMI:
            hits = hits[:1]
        if jointype in (P.JOIN_INNER, P.JOIN_LEFT, P.JOIN_FULL, P.JOIN_RIGHT, P.JOIN_SEMI):
            out += [row(o, irows[j]) for j in hits if q(o, irows[j]) is True]
        if not hits and jointype in (P.JOIN_LEFT, P.JOIN_FULL, P.JOIN_ANTI) and q(o, nul_i) is True:
            out.append(row(o, nul_i))
    if jointype in (P.JOIN_RIGHT, P.JOIN_FULL):
        out += [row(nul_o, i) for j, i in enumerate(irows) if j not in matched and q(nul_o, i) is True]
    return out


def _norm(rows):
    return sorted(tuple("~" if x is None else ("NaN" if isinstance(x, float) and math.isnan(x) else str(x)) for x in r) for r in rows)


def _rels(nf, nd, dup, key_null=0.1):
    from oracle import oracle as O
    fo = outer_rel(nf, 91, 40).set_dict_hashes(O.hashbpchar)
    do = inner_rel(nd, 92, 80, dup, unique_b=dup == "skew", key_null=key_null).set_dict_hashes(O.hashbpchar)
    return fo, do


@pytest.mark.parametrize("jointype", [P.JOIN_LEFT, P.JOIN_SEMI, P.JOIN_ANTI])
@pytest.mark.parametrize("filt", sorted(FILTERS))
@pytest.mark.parametrize("dup", [1, 3, "skew"])
def test_join_filters_against_a_nested_loop(jointype, filt, dup):
    """NULL keys and NULL filter inputs on both sides, NaNs, 1 / 3 / all build rows per key"""
    from oracle import oracle as O
    fo, do = _rels(300, 120, dup)
    got = O.execute(join_plan(jointype, fo, do, FILTERS[filt]()), [[fo, do]]).rows
    want = brute(jointype, fo, do, PY_FILTERS[filt])
    assert _norm(got) == _norm(want)
    assert len(want) > 0


@pytest.mark.parametrize("jointype,with_filter", [(jt, wf) for jt in sorted(QUALS) for wf in (False, True)
                                                  if not (wf and jt not in (P.JOIN_LEFT, P.JOIN_SEMI, P.JOIN_ANTI))])
@pytest.mark.parametrize("nf,nd", [(300, 120), (0, 120), (300, 0)])
def test_plan_qual_on_every_join_type(jointype, with_filter, nf, nd):
    """the plan's qual over joined and NULL-extended rows (NULL inner values make it NULL, which drops the row)"""
    from oracle import oracle as O
    fo, do = _rels(nf, nd, 3, key_null=0.0 if jointype == P.JOIN_LASJ_NOTIN else 0.1)
    plan = join_plan(jointype, fo, do, FILTERS["lt"]() if with_filter else (), QUALS[jointype]())
    got = O.execute(plan, [[fo, do]]).rows
    want = brute(jointype, fo, do, PY_FILTERS["lt"] if with_filter else None, PY_QUALS[jointype])
    assert _norm(got) == _norm(want)
    if nf and nd:
        assert len(want) > 0


def test_not_in_with_a_null_in_the_set_returns_nothing():
    from oracle import oracle as O
    fo, do = _rels(300, 120, 3, key_null=0.1)
    plan = join_plan(P.JOIN_LASJ_NOTIN, fo, do, (), QUALS[P.JOIN_LASJ_NOTIN]())
    assert O.execute(plan, [[fo, do]]).rows == [] == brute(P.JOIN_LASJ_NOTIN, fo, do, None, PY_QUALS[P.JOIN_LASJ_NOTIN])


@pytest.mark.parametrize("sf", [0.01, 0.1])
def test_q21_oracle_against_numpy(sf):
    """the oracle runs q21_plan as the reference executor would; numpy_answer evaluates the SQL on its own"""
    from oracle import oracle as O
    rels = tpch_q21.gen_tables(sf, O.hashbpchar)
    got = [tuple(r) for r in O.execute(tpch_q21.q21_plan(), [rels]).rows]
    want = tpch_q21.numpy_answer(sf)
    assert got == want and len(want) >= 1
    if sf >= 0.1:
        assert len(want) > 10 and want[0][1] > want[-1][1]
