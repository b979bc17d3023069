"""TPC-H Q21 (suppliers who kept orders waiting) over this repository's synthetic generator.

Host-side harness code (tables, plan, an independent numpy answer); no compute on the product path.

Q21 needs columns the Q1 / Q3 / Q5 schema (tpch.SCHEMA) does not carry.  They come from the same counter-based formulas
as tpch.gen_lineitem / gen_orders, so every value is a pure function of (seed, column id, row index):

- l_receiptdate: the receipt date gen_lineitem computes (ship date + 1 + U[0, 30));
- l_commitdate: o_orderdate + U[30, 90] (column id 29, new here);
- o_orderstatus: 'F' if every line of the order has l_linestatus 'F', 'O' if every line has 'O', else 'P';
- s_name: a dictionary of 'Supplier#%09d', whose code order is the names' byte order.

    select s_name, count(*) as numwait
    from supplier, lineitem l1, orders, nation
    where s_suppkey = l1.l_suppkey and o_orderkey = l1.l_orderkey and o_orderstatus = 'F'
      and l1.l_receiptdate > l1.l_commitdate
      and exists (select * from lineitem l2 where l2.l_orderkey = l1.l_orderkey and l2.l_suppkey <> l1.l_suppkey)
      and not exists (select * from lineitem l3 where l3.l_orderkey = l1.l_orderkey and l3.l_suppkey <> l1.l_suppkey
                      and l3.l_receiptdate > l3.l_commitdate)
      and s_nationkey = n_nationkey and n_name = 'SAUDI ARABIA'
    group by s_name order by numwait desc, s_name limit 100
"""
import numpy as np

from . import plan as P
from . import tpch
from .relation import HostRelation

RT = ["lineitem", "orders", "supplier", "nation"]
SCHEMA = {
    "lineitem": [("l_orderkey", P.INT8), ("l_suppkey", P.INT4), ("l_commitdate", P.DATE), ("l_receiptdate", P.DATE)],
    "orders": [("o_orderkey", P.INT8), ("o_orderstatus", P.BPCHAR1)],
    "supplier": [("s_suppkey", P.INT4), ("s_nationkey", P.INT4), ("s_name", P.DICT32)],
    "nation": [("n_nationkey", P.INT4), ("n_name", P.DICT8)],
}
COMMIT_COL = 29
SAUDI_ARABIA = tpch.NATIONS.index("SAUDI ARABIA")
# the device top-N (LimitSort) takes LIMIT <= 64 and refuses Q21's LIMIT 100 (CBGPU_ERR_UNSUPPORTED), so the GPU runs of
# Q21 ask for the first 64 rows of the same order
DEVICE_LIMIT = 64


def gen_columns(sf, seed=42):
    """{table: {column: array}} for Q21 at scale factor sf, plus the supplier names"""
    sz = tpch.sizes(sf)
    li = tpch.gen_lineitem(seed, sz["lineitem"], sz["supplier"], sz["part"])
    j = np.arange(sz["lineitem"], dtype=np.int64)
    oidx = (j // 28) * 7 + tpch._LINE_OFF[j % 28]
    odate = tpch.STARTDATE + (tpch._u(seed, 12, oidx) % np.uint64(tpch.ORDER_DATE_SPAN)).astype(np.int64)
    receipt = li["l_shipdate"].astype(np.int64) + 1 + (tpch._u(seed, 26, j) % np.uint64(30)).astype(np.int64)
    commit = odate + 30 + (tpch._u(seed, COMMIT_COL, j) % np.uint64(61)).astype(np.int64)
    n_orders = sz["orders"]
    inside = oidx < n_orders
    n_f = np.bincount(oidx[inside], weights=(li["l_linestatus"][inside] == ord("F")), minlength=n_orders)
    n_all = np.bincount(oidx[inside], minlength=n_orders)
    status = np.where(n_f == n_all, ord("F"), np.where(n_f == 0, ord("O"), ord("P"))).astype(np.uint8)
    supp = tpch.gen_supplier(seed, sz["supplier"])
    nation, _ = tpch.gen_nation_region()
    names = ["Supplier#%09d" % (k + 1) for k in range(sz["supplier"])]
    return {
        "lineitem": {"l_orderkey": li["l_orderkey"], "l_suppkey": li["l_suppkey"], "l_commitdate": commit.astype(np.int32),
                     "l_receiptdate": receipt.astype(np.int32)},
        "orders": {"o_orderkey": tpch.order_key(np.arange(n_orders)), "o_orderstatus": status},
        "supplier": {"s_suppkey": supp["s_suppkey"], "s_nationkey": supp["s_nationkey"],
                     "s_name": np.arange(sz["supplier"], dtype=np.int32)},
        "nation": {"n_nationkey": nation["n_nationkey"], "n_name": nation["n_name"]},
    }, names


def gen_tables(sf, hashfn, seed=42):
    """Q21's range table (RT order) as host relations, dictionary hashes through `hashfn`"""
    cols, names = gen_columns(sf, seed)
    texts = {"s_name": names, "n_name": tpch.NATIONS}
    rels = []
    for t in RT:
        cn = [c for c, _ in SCHEMA[t]]
        rels.append(HostRelation(t, cn, [ty for _, ty in SCHEMA[t]], [cols[t][c] for c in cn],
                                 dict_texts=[texts.get(c) for c in cn]).set_dict_hashes(hashfn))
    return rels


def _svar(rel, col):
    relid = RT.index(rel) + 1
    names = [c for c, _ in SCHEMA[rel]]
    return P.Var(relid, names.index(col) + 1, SCHEMA[rel][names.index(col)][1])


def _scan(rel, cols, quals=()):
    return P.SeqScan(RT.index(rel) + 1, [(c, _svar(rel, c)) for c in cols], quals)


def _late():
    return [P.OpExpr(P.OP_GT, _svar("lineitem", "l_receiptdate"), _svar("lineitem", "l_commitdate"))]


def q21_plan(nation_code=SAUDI_ARABIA, limit=100):
    """The reference planner's shape for Q21 on one segment:
    Limit <- Sort (numwait desc, s_name) <- HashAggregate (s_name)
      <- Hash Anti Join (l3.l_orderkey = l1.l_orderkey; Join Filter: l3.l_suppkey <> l1.l_suppkey)
           <- Hash Semi Join (l2.l_orderkey = l1.l_orderkey; Join Filter: l2.l_suppkey <> l1.l_suppkey)
                <- Hash Join (o_orderkey = l1.l_orderkey)
                     <- Hash Join (s_suppkey = l1.l_suppkey)
                          <- Seq Scan lineitem l1 (l_receiptdate > l_commitdate)
                          <- Hash <- Hash Join (s_nationkey = n_nationkey) <- Seq Scan supplier, Hash <- Seq Scan nation (n_name)
                     <- Hash <- Seq Scan orders (o_orderstatus = 'F')
                <- Hash <- Seq Scan lineitem l2
           <- Hash <- Seq Scan lineitem l3 (l_receiptdate > l_commitdate)"""
    nat = _scan("nation", ["n_nationkey"], [P.OpExpr(P.OP_EQ, _svar("nation", "n_name"), P.Const(P.DICT8, nation_code))])
    supp = _scan("supplier", ["s_suppkey", "s_nationkey", "s_name"])
    sn = P.HashJoin(P.JOIN_INNER, supp, P.Hash(nat, [P.out_var(nat, 1)]), [P.out_var(supp, 2)],
                    [("s_suppkey", P.out_var(supp, 1)), ("s_name", P.out_var(supp, 3))])
    l1 = _scan("lineitem", ["l_orderkey", "l_suppkey"], _late())
    j1 = P.HashJoin(P.JOIN_INNER, l1, P.Hash(sn, [P.out_var(sn, 1)]), [P.out_var(l1, 2)],
                    [("l_orderkey", P.out_var(l1, 1)), ("l_suppkey", P.out_var(l1, 2)), ("s_name", P.InnerVar(2, P.DICT32))])
    orders = _scan("orders", ["o_orderkey"], [P.OpExpr(P.OP_EQ, _svar("orders", "o_orderstatus"), P.Const(P.BPCHAR1, ord("F")))])
    j2 = P.HashJoin(P.JOIN_INNER, j1, P.Hash(orders, [P.out_var(orders, 1)]), [P.out_var(j1, 1)],
                    [("l_orderkey", P.out_var(j1, 1)), ("l_suppkey", P.out_var(j1, 2)), ("s_name", P.out_var(j1, 3))])
    l2 = _scan("lineitem", ["l_orderkey", "l_suppkey"])
    j3 = P.HashJoin(P.JOIN_SEMI, j2, P.Hash(l2, [P.out_var(l2, 1)]), [P.out_var(j2, 1)],
                    [("l_orderkey", P.out_var(j2, 1)), ("l_suppkey", P.out_var(j2, 2)), ("s_name", P.out_var(j2, 3))],
                    joinquals=[P.OpExpr(P.OP_NE, P.InnerVar(2, P.INT4), P.out_var(j2, 2))])
    l3 = _scan("lineitem", ["l_orderkey", "l_suppkey"], _late())
    j4 = P.HashJoin(P.JOIN_ANTI, j3, P.Hash(l3, [P.out_var(l3, 1)]), [P.out_var(j3, 1)], [("s_name", P.out_var(j3, 3))],
                    joinquals=[P.OpExpr(P.OP_NE, P.InnerVar(2, P.INT4), P.out_var(j3, 2))])
    agg = P.Agg(j4, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [1], [("s_name", P.out_var(j4, 1)), ("numwait", P.Aggref(P.AGG_COUNT_STAR))],
                num_groups=1000)
    return P.LimitSort(agg, [(2, True), (1, False)], limit)


def numpy_answer(sf, nation_code=SAUDI_ARABIA, limit=100, seed=42):
    """[(s_name code, numwait)] in the query's order, evaluated with numpy from the SQL (no code shared with the executor or
    the oracle).  Per order: the smallest and largest supplier over all its lines and over its late lines; a line has another
    supplier in its order exactly when one of those differs from its own."""
    cols, _ = gen_columns(sf, seed)
    li, od, su = cols["lineitem"], cols["orders"], cols["supplier"]
    okey, skey = li["l_orderkey"], li["l_suppkey"].astype(np.int64)
    late = li["l_receiptdate"] > li["l_commitdate"]
    uk, o = np.unique(okey, return_inverse=True)
    big = np.iinfo(np.int64).max
    lo_all, hi_all = np.full(len(uk), big), np.full(len(uk), -1)
    np.minimum.at(lo_all, o, skey)
    np.maximum.at(hi_all, o, skey)
    lo_late, hi_late = np.full(len(uk), big), np.full(len(uk), -1)
    np.minimum.at(lo_late, o[late], skey[late])
    np.maximum.at(hi_late, o[late], skey[late])
    exists_other = (lo_all[o] != skey) | (hi_all[o] != skey)
    late_other = (hi_late[o] >= 0) & ((lo_late[o] != skey) | (hi_late[o] != skey))
    pos = np.minimum(np.searchsorted(od["o_orderkey"], okey), len(od["o_orderkey"]) - 1)    # order keys ascend
    status_f = (od["o_orderkey"][pos] == okey) & (od["o_orderstatus"][pos] == ord("F"))
    in_nation = su["s_nationkey"][skey - 1] == nation_code     # s_suppkey = row + 1
    keep = late & status_f & in_nation & exists_other & ~late_other
    counts = np.bincount(skey[keep] - 1, minlength=len(su["s_suppkey"]))
    codes = np.nonzero(counts)[0]
    order = np.lexsort((codes, -counts[codes]))
    return [(int(codes[k]), int(counts[codes[k]])) for k in order[:limit]]
