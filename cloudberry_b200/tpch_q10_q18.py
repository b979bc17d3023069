"""TPC-H Q10 (returned-item reporting) and Q18 (large-volume customers) over this repository's synthetic generator.

Host-side harness code (tables, plans, independent numpy answers); no compute on the product path.

Both queries group by more than four columns (Q10 by seven, Q18 by five).  They need columns the Q1 / Q3 / Q5 schema
(tpch.SCHEMA) does not carry; those come from the same counter-based formulas as tpch.gen_lineitem / gen_customer, so every
value is a pure function of (seed, column id, row index):

- c_name: 'Customer#%09d' of c_custkey, a dictionary whose code is the customer's row (code order = byte order);
- c_acctbal: numeric(15,2) in [-999.99, 9999.99], U[0, 1099999) - 99999 cents (column id 33);
- c_phone: char(15) 'CC-AAA-BBB-CCCC', country code c_nationkey + 10 (TPC-H 4.2.2.9), the rest from column id 34; a dictionary
  with one entry per customer, code = row;
- c_address: one of ADDRESSES deterministic varchar strings, picked by column id 35;
- c_comment: one of COMMENTS deterministic varchar strings, picked by column id 36;
- o_totalprice: numeric(15,2), the sum over the order's lines of l_extendedprice * (1 + l_tax) * (1 - l_discount), each line
  rounded half up to cents (TPC-H 4.2.3 defines o_totalprice from the lines the same way);
- l_tax: as tpch.gen_lineitem makes it.

The synthetic lineitem gives order k exactly k mod 7 + 1 lines of quantity U[1, 50], so at most 350 per order and few above
300: Q18's threshold is a parameter (q18_plan, q18_numpy_answer) so that small scale factors select something.

    -- Q10
    select c_custkey, c_name, sum(l_extendedprice * (1 - l_discount)) as revenue, c_acctbal, n_name, c_address, c_phone,
           c_comment
    from customer, orders, lineitem, nation
    where c_custkey = o_custkey and l_orderkey = o_orderkey and o_orderdate >= date '1993-10-01'
      and o_orderdate < date '1993-10-01' + interval '3' month and l_returnflag = 'R' and c_nationkey = n_nationkey
    group by c_custkey, c_name, c_acctbal, c_phone, n_name, c_address, c_comment
    order by revenue desc limit 20

    -- Q18
    select c_name, c_custkey, o_orderkey, o_orderdate, o_totalprice, sum(l_quantity)
    from customer, orders, lineitem
    where o_orderkey in (select l_orderkey from lineitem group by l_orderkey having sum(l_quantity) > 300)
      and c_custkey = o_custkey and o_orderkey = l_orderkey
    group by c_name, c_custkey, o_orderkey, o_orderdate, o_totalprice
    order by o_totalprice desc, o_orderdate limit 100

Each plan's sort ends with one more key (Q10: c_custkey, Q18: o_orderkey) that the query leaves open, so that rows whose sort
keys tie have one order and the device and numpy can be compared row by row.
"""
import numpy as np

from . import plan as P
from . import tpch
from .relation import HostRelation

RT = ["lineitem", "orders", "customer", "nation"]
SCHEMA = {
    "lineitem": [("l_orderkey", P.INT8), ("l_quantity", P.NUMERIC), ("l_extendedprice", P.NUMERIC), ("l_discount", P.NUMERIC),
                 ("l_returnflag", P.BPCHAR1)],
    "orders": [("o_orderkey", P.INT8), ("o_custkey", P.INT4), ("o_orderdate", P.DATE), ("o_totalprice", P.NUMERIC)],
    "customer": [("c_custkey", P.INT4), ("c_name", P.DICT32), ("c_address", P.DICT32), ("c_nationkey", P.INT4),
                 ("c_phone", P.DICT32), ("c_acctbal", P.NUMERIC), ("c_comment", P.DICT32)],
    "nation": [("n_nationkey", P.INT4), ("n_name", P.DICT8)],
}
# how the reference distributes them (rpt_tpch.source: DISTRIBUTED BY / REPLICATED)
DIST_KEY = {"lineitem": "l_orderkey", "orders": "o_orderkey", "customer": None, "nation": None}
ADDRESSES = ["%d %s %s" % (100 + 37 * k, ["Oak", "Pine", "Maple", "Cedar", "Elm", "Birch", "Ash", "Willow"][k % 8],
                           ["Street", "Avenue", "Road", "Lane", "Way"][(k // 8) % 5]) for k in range(1000)]
COMMENTS = ["%s %s %s" % (["carefully", "quickly", "slyly", "blithely", "furiously", "fluffily", "boldly"][k % 7],
                          ["final", "regular", "express", "ironic", "pending", "special", "even", "unusual"][(k // 7) % 8],
                          ["deposits", "requests", "accounts", "packages", "instructions", "foxes", "theodolites",
                           "pinto beans", "asymptotes"][(k // 56) % 9]) + (" #%d" % (k // 504) if k >= 504 else "")
            for k in range(500)]
Q10_DATE_LO = tpch.date_to_days(1993, 10, 1)
Q10_DATE_HI = tpch.date_to_days(1994, 1, 1)
ACCTBAL_COL, PHONE_COL, ADDRESS_COL, COMMENT_COL = 33, 34, 35, 36


def gen_columns(sf, seed=42):
    """{table: {column: array}} for Q10 / Q18 at scale factor sf, plus the dictionaries {column: [text]}"""
    sz = tpch.sizes(sf)
    li = tpch.gen_lineitem(seed, sz["lineitem"], sz["supplier"], sz["part"])
    n_orders, n_cust = sz["orders"], sz["customer"]
    od = tpch.gen_orders(seed, n_orders, n_cust)
    j = np.arange(sz["lineitem"], dtype=np.int64)
    oidx = (j // 28) * 7 + tpch._LINE_OFF[j % 28]
    inside = oidx < n_orders
    line_cents = (li["l_extendedprice"] * (100 + li["l_tax"]) * (100 - li["l_discount"]) + 5000) // 10000
    # per-order sums below 2^53: float64 bincount weights add them exactly
    total = np.rint(np.bincount(oidx[inside], weights=line_cents[inside], minlength=n_orders)).astype(np.int64)
    cu = tpch.gen_customer(seed, n_cust)
    i = np.arange(n_cust, dtype=np.int64)
    acctbal = (tpch._u(seed, ACCTBAL_COL, i) % np.uint64(1099999)).astype(np.int64) - 99999
    ph = tpch._u(seed, PHONE_COL, i)
    a, b, c = ph % np.uint64(900) + np.uint64(100), (ph >> np.uint64(16)) % np.uint64(900) + np.uint64(100), \
        (ph >> np.uint64(32)) % np.uint64(9000) + np.uint64(1000)
    phones = ["%02d-%03d-%03d-%04d" % (n + 10, x, y, z) for n, x, y, z in zip(cu["c_nationkey"].tolist(), a.tolist(), b.tolist(),
                                                                                 c.tolist())]
    nation, _ = tpch.gen_nation_region()
    cols = {
        "lineitem": {"l_orderkey": li["l_orderkey"], "l_quantity": li["l_quantity"], "l_extendedprice": li["l_extendedprice"],
                     "l_discount": li["l_discount"], "l_returnflag": li["l_returnflag"]},
        "orders": {"o_orderkey": od["o_orderkey"], "o_custkey": od["o_custkey"], "o_orderdate": od["o_orderdate"],
                   "o_totalprice": total},
        "customer": {"c_custkey": cu["c_custkey"], "c_name": i.astype(np.int32),
                     "c_address": (tpch._u(seed, ADDRESS_COL, i) % np.uint64(len(ADDRESSES))).astype(np.int32),
                     "c_nationkey": cu["c_nationkey"], "c_phone": i.astype(np.int32), "c_acctbal": acctbal,
                     "c_comment": (tpch._u(seed, COMMENT_COL, i) % np.uint64(len(COMMENTS))).astype(np.int32)},
        "nation": {"n_nationkey": nation["n_nationkey"], "n_name": nation["n_name"]},
    }
    texts = {"c_name": ["Customer#%09d" % (k + 1) for k in range(n_cust)], "c_address": ADDRESSES, "c_phone": phones,
             "c_comment": COMMENTS, "n_name": tpch.NATIONS}
    return cols, texts


def gen_tables(sf, hashfn, seed=42):
    """the range table (RT order) as host relations, dictionary hashes through `hashfn`"""
    cols, texts = gen_columns(sf, seed)
    rels = []
    for t in RT:
        cn = [c for c, _ in SCHEMA[t]]
        rels.append(HostRelation(t, cn, [ty for _, ty in SCHEMA[t]], [cols[t][c] for c in cn],
                                 dict_texts=[texts.get(c) for c in cn]).set_dict_hashes(hashfn))
    return rels


def _svar(rel, col):
    relid = RT.index(rel) + 1
    names = [c for c, _ in SCHEMA[rel]]
    t = SCHEMA[rel][names.index(col)][1]
    return P.Var(relid, names.index(col) + 1, t, 2 if t == P.NUMERIC else 0)


def _scan(rel, cols, quals=()):
    return P.SeqScan(RT.index(rel) + 1, [(c, _svar(rel, c)) for c in cols], quals)


def _top(agg, keys, limit, nsegs):
    """Limit <- Sort on one segment; with several, each segment's Limit <- Sort under a Gather and the same on top of it"""
    top = P.LimitSort(agg, keys, limit)
    if nsegs == 1:
        return top
    return P.LimitSort(P.Motion(top, P.MOTIONTYPE_GATHER), keys, limit)


def q10_plan(limit=20, date_lo=Q10_DATE_LO, date_hi=Q10_DATE_HI, sf=1):
    """The reference planner's shape for Q10 on one segment, its group estimate for scale factor sf (the customers with a
    returned line in the quarter: 28 % of them in this data, estimated as 30 %):
    Limit <- Sort (revenue desc, c_custkey)
      <- HashAggregate (c_custkey, c_name, c_acctbal, c_phone, n_name, c_address, c_comment)
        <- Hash Join (l_orderkey = o_orderkey)
             <- Seq Scan lineitem (l_returnflag = 'R')
             <- Hash <- Hash Join (o_custkey = c_custkey)
                          <- Seq Scan orders (o_orderdate in [date_lo, date_hi))
                          <- Hash <- Hash Join (c_nationkey = n_nationkey) <- Seq Scan customer, Hash <- Seq Scan nation"""
    nat = _scan("nation", ["n_nationkey", "n_name"])
    cust = _scan("customer", ["c_custkey", "c_name", "c_acctbal", "c_phone", "c_address", "c_comment", "c_nationkey"])
    cn = P.HashJoin(P.JOIN_INNER, cust, P.Hash(nat, [P.out_var(nat, 1)]), [P.out_var(cust, 7)],
                    [("c_custkey", P.out_var(cust, 1)), ("c_name", P.out_var(cust, 2)), ("c_acctbal", P.out_var(cust, 3)),
                     ("c_phone", P.out_var(cust, 4)), ("n_name", P.InnerVar(2, P.DICT8)), ("c_address", P.out_var(cust, 5)),
                     ("c_comment", P.out_var(cust, 6))])
    orders = _scan("orders", ["o_orderkey", "o_custkey"],
                   [P.OpExpr(P.OP_GE, _svar("orders", "o_orderdate"), P.Const(P.DATE, date_lo)),
                    P.OpExpr(P.OP_LT, _svar("orders", "o_orderdate"), P.Const(P.DATE, date_hi))])
    oc = P.HashJoin(P.JOIN_INNER, orders, P.Hash(cn, [P.out_var(cn, 1)]), [P.out_var(orders, 2)],
                    [("o_orderkey", P.out_var(orders, 1))] +
                    [(name, P.InnerVar(k + 1, *P.out_type(cn, k + 1))) for k, name in
                     enumerate(["c_custkey", "c_name", "c_acctbal", "c_phone", "n_name", "c_address", "c_comment"])])
    li = _scan("lineitem", ["l_orderkey", "l_extendedprice", "l_discount"],
               [P.OpExpr(P.OP_EQ, _svar("lineitem", "l_returnflag"), P.Const(P.BPCHAR1, ord("R")))])
    j = P.HashJoin(P.JOIN_INNER, li, P.Hash(oc, [P.out_var(oc, 1)]), [P.out_var(li, 1)],
                   [(name, P.InnerVar(k + 2, *P.out_type(oc, k + 2))) for k, name in
                    enumerate(["c_custkey", "c_name", "c_acctbal", "c_phone", "n_name", "c_address", "c_comment"])] +
                   [("l_extendedprice", P.out_var(li, 2)), ("l_discount", P.out_var(li, 3))])
    v = lambda k: P.out_var(j, k)       # noqa: E731
    rev = P.OpExpr(P.OP_MUL, v(8), P.OpExpr(P.OP_SUB, P.NumericConst("1"), v(9)))
    agg = P.Agg(j, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1, 2, 3, 4, 5, 6, 7],
                [("c_custkey", v(1)), ("c_name", v(2)), ("revenue", P.Aggref(P.AGG_SUM, rev)), ("c_acctbal", v(3)),
                 ("n_name", v(5)), ("c_address", v(6)), ("c_phone", v(4)), ("c_comment", v(7))],
                num_groups=max(tpch.sizes(sf)["customer"] * 3 // 10, 1))
    return P.LimitSort(agg, [(3, True), (1, False)], limit)


def q18_subquery(threshold=300, sf=1, having=True):
    """Q18's IN subquery: HashAggregate (l_orderkey) [Filter: sum(l_quantity) > threshold] <- Seq Scan lineitem, one group per
    order; without `having` the same aggregate passes every group on"""
    scan = _scan("lineitem", ["l_orderkey", "l_quantity"])
    quals = [P.OpExpr(P.OP_GT, P.Aggref(P.AGG_SUM, P.out_var(scan, 2)), P.NumericConst(str(threshold)))] if having else []
    return P.Agg(scan, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("l_orderkey", P.out_var(scan, 1))],
                 num_groups=tpch.sizes(sf)["orders"], quals=quals)


def q18_plan(threshold=300, limit=100, nsegs=1, sf=1):
    """The reference planner's shape for Q18 (the IN subquery's groups are unique on l_orderkey, so it joins as an inner join),
    its group estimates for scale factor sf (the subquery: one group per order; the outer aggregate: the orders that pass
    HAVING, under 1 % of them in this data at any threshold from 250 up):
    Limit <- Sort (o_totalprice desc, o_orderdate, o_orderkey)
      <- HashAggregate (c_name, c_custkey, o_orderkey, o_orderdate, o_totalprice)
        <- Hash Join (l_orderkey = o_orderkey)
             <- Seq Scan lineitem
             <- Hash <- Hash Join (o_custkey = c_custkey)
                          <- Hash Join (o_orderkey = l_orderkey)
                               <- Seq Scan orders
                               <- Hash <- HashAggregate (l_orderkey) Filter: sum(l_quantity) > threshold <- Seq Scan lineitem
                          <- Hash <- Seq Scan customer
    lineitem and orders are co-located on the order key and customer is replicated, so on nsegs > 1 segments every join and
    the aggregation (its groups contain o_orderkey) stay local: each segment's Limit <- Sort goes up a Gather."""
    sub = q18_subquery(threshold, sf)
    orders = _scan("orders", ["o_orderkey", "o_custkey", "o_orderdate", "o_totalprice"])
    os_ = P.HashJoin(P.JOIN_INNER, orders, P.Hash(sub, [P.out_var(sub, 1)]), [P.out_var(orders, 1)],
                     [("o_orderkey", P.out_var(orders, 1)), ("o_custkey", P.out_var(orders, 2)),
                      ("o_orderdate", P.out_var(orders, 3)), ("o_totalprice", P.out_var(orders, 4))])
    cust = _scan("customer", ["c_custkey", "c_name"])
    oc = P.HashJoin(P.JOIN_INNER, os_, P.Hash(cust, [P.out_var(cust, 1)]), [P.out_var(os_, 2)],
                    [("c_name", P.InnerVar(2, P.DICT32)), ("c_custkey", P.InnerVar(1, P.INT4)), ("o_orderkey", P.out_var(os_, 1)),
                     ("o_orderdate", P.out_var(os_, 3)), ("o_totalprice", P.out_var(os_, 4))])
    li = _scan("lineitem", ["l_orderkey", "l_quantity"])
    j = P.HashJoin(P.JOIN_INNER, li, P.Hash(oc, [P.out_var(oc, 3)]), [P.out_var(li, 1)],
                   [(name, P.InnerVar(k + 1, *P.out_type(oc, k + 1))) for k, name in
                    enumerate(["c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice"])] +
                   [("l_quantity", P.out_var(li, 2))])
    v = lambda k: P.out_var(j, k)       # noqa: E731
    agg = P.Agg(j, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1, 2, 3, 4, 5],
                [("c_name", v(1)), ("c_custkey", v(2)), ("o_orderkey", v(3)), ("o_orderdate", v(4)), ("o_totalprice", v(5)),
                 ("sum", P.Aggref(P.AGG_SUM, v(6)))], num_groups=max(tpch.sizes(sf)["orders"] // 100, 1))
    return _top(agg, [(5, True), (4, False), (3, False)], limit, nsegs)


def numeric_text(v, dscale):
    """a scaled integer as numeric_out prints it at display scale dscale"""
    v = int(v)
    if dscale == 0:
        return str(v)
    s = "%0*d" % (dscale + 1, abs(v))
    return ("-" if v < 0 else "") + s[:-dscale] + "." + s[-dscale:]


def q10_numpy_answer(sf, limit=20, date_lo=Q10_DATE_LO, date_hi=Q10_DATE_HI, seed=42):
    """Q10's rows in the plan's order, evaluated with numpy from the SQL (no code shared with the executor or the oracle):
    (c_custkey, c_name code, revenue, c_acctbal, n_name code, c_address code, c_phone code, c_comment code), numerics as text"""
    cols, _ = gen_columns(sf, seed)
    li, od, cu = cols["lineitem"], cols["orders"], cols["customer"]
    pos = np.minimum(np.searchsorted(od["o_orderkey"], li["l_orderkey"]), len(od["o_orderkey"]) - 1)   # order keys ascend
    keep = (od["o_orderkey"][pos] == li["l_orderkey"]) & (li["l_returnflag"] == ord("R"))
    d = od["o_orderdate"][pos]
    keep &= (d >= date_lo) & (d < date_hi)
    cust = od["o_custkey"][pos][keep].astype(np.int64) - 1            # c_custkey = row + 1
    rev = (li["l_extendedprice"] * (100 - li["l_discount"]))[keep]    # scale 4
    total = np.rint(np.bincount(cust, weights=rev, minlength=len(cu["c_custkey"]))).astype(np.int64)   # exact below 2^53
    rows = np.unique(cust)
    order = np.lexsort((rows, -total[rows]))
    return [(int(cu["c_custkey"][r]), int(cu["c_name"][r]), numeric_text(total[r], 4), numeric_text(cu["c_acctbal"][r], 2),
             int(cu["c_nationkey"][r]), int(cu["c_address"][r]), int(cu["c_phone"][r]), int(cu["c_comment"][r]))
            for r in rows[order[:limit]]]


def q18_numpy_answer(sf, threshold=300, limit=100, seed=42):
    """Q18's rows in the plan's order, evaluated with numpy from the SQL: (c_name code, c_custkey, o_orderkey, o_orderdate,
    o_totalprice, sum(l_quantity)), numerics as text"""
    cols, _ = gen_columns(sf, seed)
    li, od, cu = cols["lineitem"], cols["orders"], cols["customer"]
    uk, inv = np.unique(li["l_orderkey"], return_inverse=True)
    qty = np.rint(np.bincount(inv, weights=li["l_quantity"], minlength=len(uk))).astype(np.int64)
    big = uk[qty > threshold * 100]                                    # l_quantity is scaled by 100
    pos = np.searchsorted(od["o_orderkey"], big)
    ok = pos < len(od["o_orderkey"])
    ok[ok] = od["o_orderkey"][pos[ok]] == big[ok]
    pos, bq = pos[ok], qty[qty > threshold * 100][ok]
    price, date, okey = od["o_totalprice"][pos], od["o_orderdate"][pos], od["o_orderkey"][pos]
    order = np.lexsort((okey, date, -price))[:limit]
    c = od["o_custkey"][pos].astype(np.int64) - 1
    return [(int(cu["c_name"][c[k]]), int(cu["c_custkey"][c[k]]), int(okey[k]), int(date[k]), numeric_text(price[k], 2),
             numeric_text(bq[k], 2)) for k in order]
