"""ctypes mirror of include/cb_plan.h plus small constructors for plan trees.

The structs mirror the reference's planner output (src/include/nodes/plannodes.h:263-337 Plan,
:1193 HashJoin, :1342 Agg, :1551 Hash, :1651 Motion; src/include/nodes/primnodes.h Var / Const /
OpExpr / BoolExpr / Aggref / TargetEntry), so a test builds the tree the reference planner emits
for a query (e.g. expected/aggregates.out:3313-3328) and hands the same tree to the GPU executor
and to the CPU oracle.

Host-side glue only: no compute happens here.
"""
import ctypes as C

# ---- CbTypeId ----
INT4, INT8, DATE, NUMERIC, BPCHAR1, DICT8, DICT32, FLOAT8, BOOL, NUMERIC128, TEXT = range(1, 12)
TYPE_WIDTH = {INT4: 4, INT8: 8, DATE: 4, NUMERIC: 8, BPCHAR1: 1, DICT8: 1, DICT32: 4, FLOAT8: 8, BOOL: 1, NUMERIC128: 16}
TYPE_NAME = {INT4: "int4", INT8: "int8", DATE: "date", NUMERIC: "numeric", BPCHAR1: "bpchar1", DICT8: "dict8",
             DICT32: "dict32", FLOAT8: "float8", BOOL: "bool", NUMERIC128: "numeric128"}

# ---- CbNodeTag ----
T_SeqScan, T_Hash, T_HashJoin, T_Agg, T_Motion, T_LimitSort = range(100, 106)
T_Var, T_Const, T_OpExpr, T_BoolExpr, T_Aggref, T_ScalarArrayOpExpr = range(200, 206)

INNER_VAR, OUTER_VAR = 65000, 65001

OP_ADD, OP_SUB, OP_MUL = 1, 2, 3
OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE = 10, 11, 12, 13, 14, 15
OP_LIKE, OP_NOTLIKE = 20, 21
AND_EXPR, OR_EXPR, NOT_EXPR = 0, 1, 2
AGG_COUNT_STAR, AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX = 1, 2, 3, 4, 5, 6
JOIN_INNER, JOIN_LEFT, JOIN_FULL, JOIN_RIGHT, JOIN_SEMI, JOIN_ANTI, JOIN_LASJ_NOTIN = range(7)
AGG_PLAIN, AGG_SORTED, AGG_HASHED, AGG_MIXED = range(4)
AGGSPLIT_SIMPLE, AGGSPLIT_INITIAL_SERIAL, AGGSPLIT_FINAL_DESERIAL = range(3)
MOTIONTYPE_GATHER, MOTIONTYPE_GATHER_SINGLE, MOTIONTYPE_HASH, MOTIONTYPE_BROADCAST = range(4)


class CbExpr(C.Structure):
    pass


CbExpr._fields_ = [
    ("tag", C.c_int), ("restype", C.c_int), ("dscale", C.c_int32),
    ("varno", C.c_int32), ("varattno", C.c_int32),
    ("constval", C.c_int64), ("constisnull", C.c_bool),
    ("op", C.c_int32), ("nargs", C.c_int32), ("args", C.POINTER(C.POINTER(CbExpr))),
    ("conststr", C.c_char_p), ("constlen", C.c_int32), ("useOr", C.c_bool),
]


class CbTargetEntry(C.Structure):
    _fields_ = [("expr", C.POINTER(CbExpr)), ("resno", C.c_int32), ("resname", C.c_char_p)]


class CbPlan(C.Structure):
    pass


CbPlan._fields_ = [
    ("type", C.c_int), ("plan_node_id", C.c_int32), ("plan_rows", C.c_double),
    ("ntargets", C.c_int32), ("targetlist", C.POINTER(CbTargetEntry)),
    ("nquals", C.c_int32), ("qual", C.POINTER(C.POINTER(CbExpr))),
    ("lefttree", C.POINTER(CbPlan)), ("righttree", C.POINTER(CbPlan)),
]


class CbSeqScan(C.Structure):
    _fields_ = [("plan", CbPlan), ("scanrelid", C.c_int32)]


class CbHash(C.Structure):
    _fields_ = [("plan", CbPlan), ("nhashkeys", C.c_int32), ("hashkeys", C.POINTER(C.POINTER(CbExpr)))]


class CbHashJoin(C.Structure):
    _fields_ = [("plan", CbPlan), ("jointype", C.c_int), ("nhashkeys", C.c_int32),
                ("hashkeys", C.POINTER(C.POINTER(CbExpr))), ("njoinquals", C.c_int32),
                ("joinqual", C.POINTER(C.POINTER(CbExpr)))]


class CbAgg(C.Structure):
    _fields_ = [("plan", CbPlan), ("aggstrategy", C.c_int), ("aggsplit", C.c_int), ("numCols", C.c_int32),
                ("grpColIdx", C.POINTER(C.c_int32)), ("numGroups", C.c_int64), ("streaming", C.c_bool)]


class CbSortKey(C.Structure):
    _fields_ = [("attno", C.c_int32), ("descending", C.c_bool)]


class CbMotion(C.Structure):
    _fields_ = [("plan", CbPlan), ("motionType", C.c_int), ("motionID", C.c_int32), ("nhashExprs", C.c_int32),
                ("hashExprs", C.POINTER(C.POINTER(CbExpr))), ("numHashSegments", C.c_int32), ("nsortkeys", C.c_int32),
                ("sortkeys", C.POINTER(CbSortKey))]


class CbLimitSort(C.Structure):
    _fields_ = [("plan", CbPlan), ("nkeys", C.c_int32), ("keys", C.POINTER(CbSortKey)), ("limit", C.c_int64)]


# ------------------------------------------------------------------------------------------------
# constructors.  Every ctypes object created is kept alive by hanging it off its parent (_keep).
# ------------------------------------------------------------------------------------------------
def _expr_array(exprs):
    arr = (C.POINTER(CbExpr) * max(len(exprs), 1))()
    for i, e in enumerate(exprs):
        arr[i] = C.pointer(e)
    return arr


def _arith_result(op, a, b):
    """Result type / display scale rules of the reference's operators on this path
    (numeric_add/sub keep max dscale, numeric_mul sums them: utils/adt/numeric.c:2491,2567,2645)."""
    if FLOAT8 in (a.restype, b.restype):
        return FLOAT8, 0
    if op == OP_MUL:
        ds = a.dscale + b.dscale
    else:
        ds = max(a.dscale, b.dscale)
    if NUMERIC in (a.restype, b.restype):
        return NUMERIC, ds
    if INT8 in (a.restype, b.restype):
        return INT8, 0
    if DATE in (a.restype, b.restype):
        return DATE, 0
    return INT4, 0


def Var(varno, attno, typ, dscale=0):
    e = CbExpr(tag=T_Var, restype=typ, dscale=dscale, varno=varno, varattno=attno)
    e._keep = []
    return e


def OuterVar(attno, typ, dscale=0):
    return Var(OUTER_VAR, attno, typ, dscale)


def InnerVar(attno, typ, dscale=0):
    return Var(INNER_VAR, attno, typ, dscale)


def Const(typ, value, dscale=0, isnull=False):
    if typ == FLOAT8:
        import struct
        value = struct.unpack("<q", struct.pack("<d", float(value)))[0]
    e = CbExpr(tag=T_Const, restype=typ, dscale=dscale, constval=int(value), constisnull=isnull)
    e._keep = []
    return e


def NumericConst(text):
    """numeric literal -> scaled int64 constant, dscale = digits after the point."""
    neg = text.startswith("-")
    t = text.lstrip("+-")
    ip, _, fp = t.partition(".")
    v = int(ip or "0") * 10 ** len(fp) + int(fp or "0")
    return Const(NUMERIC, -v if neg else v, dscale=len(fp))


def OpExpr(op, a, b):
    if op >= OP_EQ:
        typ, ds = BOOL, 0
    else:
        typ, ds = _arith_result(op, a, b)
    e = CbExpr(tag=T_OpExpr, restype=typ, dscale=ds, op=op, nargs=2)
    e._keep = [a, b, _expr_array([a, b])]
    e.args = e._keep[2]
    return e


def TextConst(text):
    """a string literal (CB_TEXT): a LIKE pattern or an IN list element"""
    b = text if isinstance(text, bytes) else text.encode()
    e = CbExpr(tag=T_Const, restype=TEXT, conststr=b, constlen=len(b))
    e._keep = [b]
    return e


def Like(var, pattern, negate=False):
    """var LIKE 'pattern' (~~), or NOT LIKE (!~~) with negate"""
    p = pattern if isinstance(pattern, CbExpr) else TextConst(pattern)
    e = CbExpr(tag=T_OpExpr, restype=BOOL, op=OP_NOTLIKE if negate else OP_LIKE, nargs=2)
    e._keep = [var, p, _expr_array([var, p])]
    e.args = e._keep[2]
    return e


def InList(var, elems, negate=False):
    """var IN (e1, ...) = ScalarArrayOpExpr(=, useOr); NOT IN = (<>, not useOr).  Elements: CbExprs, or str (TextConst) /
    int (a Const of var's type)"""
    cs = [x if isinstance(x, CbExpr) else TextConst(x) if isinstance(x, (str, bytes)) else Const(var.restype, x, var.dscale)
          for x in elems]
    e = CbExpr(tag=T_ScalarArrayOpExpr, restype=BOOL, op=OP_NE if negate else OP_EQ, nargs=1 + len(cs), useOr=not negate)
    e._keep = [var] + cs + [_expr_array([var] + cs)]
    e.args = e._keep[-1]
    return e


def BoolExpr(boolop, *args):
    e = CbExpr(tag=T_BoolExpr, restype=BOOL, op=boolop, nargs=len(args))
    e._keep = list(args) + [_expr_array(list(args))]
    e.args = e._keep[-1]
    return e


def Aggref(fn, arg=None, restype=None, dscale=None):
    """Result types follow pg_aggregate.dat: count -> int8; sum(int4) -> int8; sum(int8) and
    sum/avg(numeric) -> numeric; avg(int) -> numeric; sum/avg(float8) -> float8; min/max -> input."""
    if restype is None:
        if fn in (AGG_COUNT_STAR, AGG_COUNT):
            restype, dscale = INT8, 0
        elif fn in (AGG_MIN, AGG_MAX):
            restype, dscale = arg.restype, arg.dscale
        elif arg.restype == FLOAT8:
            restype, dscale = FLOAT8, 0
        elif fn == AGG_SUM and arg.restype == INT4:
            restype, dscale = INT8, 0
        else:
            restype, dscale = NUMERIC, arg.dscale
    e = CbExpr(tag=T_Aggref, restype=restype, dscale=dscale or 0, op=fn, nargs=0 if arg is None else 1)
    e._keep = []
    if arg is not None:
        e._keep = [arg, _expr_array([arg])]
        e.args = e._keep[1]
    return e


_next_id = [0]


def _fill_plan(p, node_type, targets, quals, left=None, right=None, plan_rows=0.0):
    _next_id[0] += 1
    p.type = node_type
    p.plan_node_id = _next_id[0]
    p.plan_rows = plan_rows
    tl = (CbTargetEntry * max(len(targets), 1))()
    keep = []
    for i, t in enumerate(targets):
        name, expr = t if isinstance(t, tuple) else (None, t)
        tl[i].expr = C.pointer(expr)
        tl[i].resno = i + 1
        tl[i].resname = name.encode() if name else None
        keep.append(expr)
    p.ntargets = len(targets)
    p.targetlist = tl
    qa = _expr_array(list(quals))
    p.nquals = len(quals)
    p.qual = qa
    keep += [tl, qa] + list(quals)
    return keep


def plan_ptr(node):
    """POINTER(CbPlan) for any node struct (the CbPlan header is the first member)."""
    return C.cast(C.pointer(node), C.POINTER(CbPlan))


def SeqScan(scanrelid, targets, quals=(), plan_rows=0.0):
    n = CbSeqScan()
    n._keep = _fill_plan(n.plan, T_SeqScan, targets, quals, plan_rows=plan_rows)
    n.scanrelid = scanrelid
    return n


def Hash(child, hashkeys):
    n = CbHash()
    # a Hash node passes its child's tuples through: targetlist = OUTER_VARs of the child
    tl = [OuterVar(i + 1, child.plan.targetlist[i].expr.contents.restype, child.plan.targetlist[i].expr.contents.dscale)
          for i in range(child.plan.ntargets)]
    n._keep = _fill_plan(n.plan, T_Hash, tl, ())
    n.plan.lefttree = plan_ptr(child)
    ka = _expr_array(list(hashkeys))
    n.nhashkeys = len(hashkeys)
    n.hashkeys = ka
    n._keep += [child, ka] + list(hashkeys)
    return n


def HashJoin(jointype, outer, inner_hash, hashkeys, targets, joinquals=(), quals=()):
    n = CbHashJoin()
    n._keep = _fill_plan(n.plan, T_HashJoin, targets, quals)
    n.plan.lefttree = plan_ptr(outer)
    n.plan.righttree = plan_ptr(inner_hash)
    n.jointype = jointype
    ka = _expr_array(list(hashkeys))
    n.nhashkeys = len(hashkeys)
    n.hashkeys = ka
    ja = _expr_array(list(joinquals))
    n.njoinquals = len(joinquals)
    n.joinqual = ja
    n._keep += [outer, inner_hash, ka, ja] + list(hashkeys) + list(joinquals)
    return n


def Agg(child, strategy, split, grp_col_idx, targets, num_groups=0, quals=(), streaming=False):
    n = CbAgg()
    n._keep = _fill_plan(n.plan, T_Agg, targets, quals)
    n.plan.lefttree = plan_ptr(child)
    n.aggstrategy = strategy
    n.aggsplit = split
    n.numCols = len(grp_col_idx)
    ga = (C.c_int32 * max(len(grp_col_idx), 1))(*grp_col_idx)
    n.grpColIdx = ga
    n.numGroups = num_groups
    n.streaming = streaming
    n._keep += [child, ga]
    return n


def Motion(child, motion_type, hash_exprs=(), num_hash_segments=0, motion_id=None, sort_keys=()):
    """sort_keys: [(attno, descending)] - a Gather whose receiver merges the senders' sorted streams (Motion.sendSorted)"""
    n = CbMotion()
    tl = [OuterVar(i + 1, child.plan.targetlist[i].expr.contents.restype, child.plan.targetlist[i].expr.contents.dscale)
          for i in range(child.plan.ntargets)]
    n._keep = _fill_plan(n.plan, T_Motion, tl, ())
    n.plan.lefttree = plan_ptr(child)
    n.motionType = motion_type
    n.motionID = motion_id if motion_id is not None else n.plan.plan_node_id
    ha = _expr_array(list(hash_exprs))
    n.nhashExprs = len(hash_exprs)
    n.hashExprs = ha
    n.numHashSegments = num_hash_segments
    sk = (CbSortKey * max(len(sort_keys), 1))()
    for i, (attno, desc) in enumerate(sort_keys):
        sk[i].attno = attno
        sk[i].descending = bool(desc)
    n.nsortkeys = len(sort_keys)
    n.sortkeys = C.cast(sk, C.POINTER(CbSortKey))
    n._keep += [child, ha, sk] + list(hash_exprs)
    return n


def LimitSort(child, keys, limit, targets=None):
    """keys: [(attno, descending)]"""
    n = CbLimitSort()
    if targets is None:
        targets = [OuterVar(i + 1, child.plan.targetlist[i].expr.contents.restype,
                            child.plan.targetlist[i].expr.contents.dscale) for i in range(child.plan.ntargets)]
    n._keep = _fill_plan(n.plan, T_LimitSort, targets, ())
    n.plan.lefttree = plan_ptr(child)
    ka = (CbSortKey * max(len(keys), 1))()
    for i, (attno, desc) in enumerate(keys):
        ka[i].attno = attno
        ka[i].descending = desc
    n.nkeys = len(keys)
    n.keys = ka
    n.limit = limit
    n._keep += [child, ka]
    return n


def out_type(node, attno):
    """(type, dscale) of a node's output column (1-based)."""
    e = node.plan.targetlist[attno - 1].expr.contents
    return e.restype, e.dscale


def out_var(node, attno):
    t, ds = out_type(node, attno)
    return OuterVar(attno, t, ds)
