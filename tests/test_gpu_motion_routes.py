"""Where every hash Motion puts each row: CUDA executor vs the CPU oracle, row by row (-m gpu).

Where a Redistribute Motion sends a row is part of the semantics (DESIGN §2): a row on the wrong segment misses the rows it
joins with there.  A query answer does not show it: a two-stage aggregate is right under any route that is a deterministic
function of the key.  So these tests run plans whose root is the Motion (or whose top slice keeps the segment it ran on) on
an in-process cluster, and compare the multiset of (segment, row) with the oracle's, whose od_hash and jump hash are held
against the reference's cdbhash.c.  float8 values are compared by bit pattern: -0, NaN payloads and NaN signs must arrive as
they were sent.  Every table is built twice, with the oracle's and with the product's hashbpchar for the per-code hashes.

Each case names in its id the kernel that must have run the sender slice's PARTITION sink, and asserts it: k_probe_chain for
non-nullable integer, date, dictionary, char(1) and bool columns, k_pipeline_generic for float8 or nullable columns,
expression keys, N:M continuations, multi-batch joins and when forced, k_prefilter + k_probe_chain in a context that sends
every join through the prefilter pass.  The direct (peer-memory) transport is checked by tests/motion_routes_worker.py."""
import os
import struct
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

from cloudberry_b200 import capi
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import to_device
from test_gpu_join_routes import PREFILTER, _context, keyset

pytestmark = pytest.mark.gpu

PC, GEN, PF = "k_probe_chain", "k_pipeline_generic", "k_prefilter"
SINK_MATERIALIZE, SINK_PARTITION = 2, 3
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1
DICT8_TEXTS = ["v%03d" % i for i in range(256)]
DICT32_TEXTS = ["w%05d" % i for i in range(5000)]


@pytest.fixture(scope="module")
def contexts():
    made = {"plain": _context({}), "prefilter": _context(PREFILTER)}
    yield made
    for c in made.values():
        c.close()


# ---- float8 values by family: each family must take one route (hashfloat8: -0 = +0, every NaN = get_float8_nan()) ----

def _f8(bits):
    return np.array(bits, dtype=np.uint64).view(np.float64)


F8_ZEROS = [0x0000000000000000, 0x8000000000000000]
F8_NANS = [0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000, 0xFFF80000DEADBEEF,      # quiet, both signs, payloads
           0x7FF0000000000001, 0x7FF4000000000000, 0xFFF0000000000001, 0xFFF7FFFFFFFFFFFF]      # signalling, both signs
F8_OTHER = [0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF, 0x0008000000000000]


def _bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def _family(v):
    b = _bits(v)
    if (b << 1) & (2 ** 64 - 1) == 0:
        return "zero"
    if (b >> 52) & 0x7FF == 0x7FF and b & (2 ** 52 - 1):
        return "nan"
    return None


# ---- key columns: name -> (types, fn(rng, n) -> columns, nulls or None) ----

def _with_specials(special, rest, dtype):
    v = np.asarray(rest).astype(dtype)
    k = min(len(special), len(v))
    v[:k] = np.asarray(special[:k], dtype=dtype)
    return v


def _int4(rng, n, special=(INT32_MIN, INT32_MAX, -1, 0)):
    return _with_specials(list(special), rng.integers(INT32_MIN, INT32_MAX, n, endpoint=True), np.int32)


def _int8_set(name):
    def gen(rng, n):
        probe = keyset(name, 2000, max(n, 1), int(rng.integers(1 << 30)))[1][0][:n] if n else np.zeros(0, np.int64)
        return _with_specials([INT64_MIN, INT64_MAX, -1, 0, 2 ** 32, -(2 ** 32)], probe, np.int64)
    return gen


def _float8(rng, n):
    special = list(_f8(F8_ZEROS + F8_NANS + F8_OTHER))
    v = rng.normal(0, 1e6, n)
    v[: min(n, len(special))] = special[: min(n, len(special))]
    if n > 200:           # each family many times over, so that one family split over two routes shows
        idx = rng.integers(0, n, n // 10)
        v[idx] = rng.choice(np.array(special), len(idx))
    return v


KEYS = {
    "int4": ([P.INT4], lambda rng, n: [_int4(rng, n)]),
    "int8_edges": ([P.INT8], lambda rng, n: [_with_specials([INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1, -1, 0],
                                                            rng.integers(INT64_MIN, INT64_MAX, n, endpoint=True), np.int64)]),
    "int8_alias": ([P.INT8], lambda rng, n: [_int8_set("int8_alias")(rng, n)]),
    "int8_fold": ([P.INT8], lambda rng, n: [_int8_set("int8_fold")(rng, n)]),
    "date": ([P.DATE], lambda rng, n: [_with_specials([-1, 0, -40000, 40000], rng.integers(-40000, 40000, n), np.int32)]),
    "float8": ([P.FLOAT8], lambda rng, n: [_float8(rng, n)]),
    "bpchar1": ([P.BPCHAR1], lambda rng, n: [_with_specials([0x20, 0x80, 0xFF, 0x41, 0x7F], rng.integers(1, 256, n), np.uint8)]),
    "bool": ([P.BOOL], lambda rng, n: [rng.integers(0, 2, n).astype(np.uint8)]),
    "dict8": ([P.DICT8], lambda rng, n: [_with_specials([0, 127, 128, 255], rng.integers(0, 256, n), np.uint8)]),
    "dict32": ([P.DICT32], lambda rng, n: [_with_specials([0, 4999], rng.integers(0, 5000, n), np.int32)]),
    "mixed2": ([P.INT4, P.DICT8], lambda rng, n: [_int4(rng, n), rng.integers(0, 256, n).astype(np.uint8)]),
    "mixed3": ([P.INT8, P.BPCHAR1, P.DATE], lambda rng, n: [rng.integers(-2 ** 40, 2 ** 40, n), rng.integers(1, 256, n).astype(np.uint8),
                                                           rng.integers(-400, 400, n).astype(np.int32)]),
    "mixed4": ([P.BOOL, P.INT4, P.DICT32, P.INT8], lambda rng, n: [rng.integers(0, 2, n).astype(np.uint8), rng.integers(-50, 50, n).astype(np.int32),
                                                                   rng.integers(0, 5000, n).astype(np.int32), rng.integers(0, 2 ** 33, n)]),
}
NULLABLE = {"null_one": "int4,int8 keys, NULL in the first", "null_all": "int4,int8 keys, rows NULL in both"}


def table(n, keyname, seed, payload_nulls=None, float_payload=False):
    """fact(k0.., q int4 in [0, 100), v int8, g dict8[, x float8]) with the key columns of KEYS[keyname] (or the nullable sets);
    both builds (oracle hashbpchar, product hashbpchar)"""
    rng = np.random.default_rng(seed)
    nulls = []
    if keyname in NULLABLE:
        ktypes = [P.INT4, P.INT8]
        keys = [rng.integers(-1000, 1000, n).astype(np.int32), rng.integers(-2 ** 40, 2 ** 40, n)]
        n0 = (rng.random(n) < 0.2).astype(np.uint8)
        n1 = n0.copy() if keyname == "null_all" else np.zeros(n, np.uint8)
        if keyname == "null_all":
            n0 |= (rng.random(n) < 0.1).astype(np.uint8)     # some rows NULL in one key only, some in both
        nulls = [n0, n1]
    else:
        ktypes, fn = KEYS[keyname]
        keys = fn(rng, n)
        nulls = [None] * len(keys)
    nk = len(keys)
    names = ["k%d" % i for i in range(nk)] + ["q", "v", "g"] + (["x"] if float_payload else [])
    types = list(ktypes) + [P.INT4, P.INT8, P.DICT8] + ([P.FLOAT8] if float_payload else [])
    cols = list(keys) + [rng.integers(0, 100, n).astype(np.int32), rng.integers(-10 ** 12, 10 ** 12, n),
                         rng.integers(0, 256, n).astype(np.uint8)] + ([_float8(rng, n)] if float_payload else [])
    nulls = nulls + [None, payload_nulls, None] + ([None] if float_payload else [])
    texts = [DICT8_TEXTS if t == P.DICT8 else DICT32_TEXTS if t == P.DICT32 else None for t in types]

    def mk():
        return HostRelation("fact", names, types, cols, nulls=nulls, dict_texts=texts)
    from oracle import oracle as O
    return mk().set_dict_hashes(O.hashbpchar), mk().set_dict_hashes(capi.hashbpchar)


def dim(n, seed, dup=1, kmax=1000):
    """dim(dk int4 over [0, kmax), c dict8 of 256 entries, w int8): dk unique (dup=1) or each key dup times (N:M)"""
    rng = np.random.default_rng(seed)
    keys = np.repeat(rng.permutation(kmax)[: n // dup], dup).astype(np.int32)
    m = len(keys)

    def mk():
        return HostRelation("dim", ["dk", "c", "w"], [P.INT4, P.DICT8, P.INT8],
                            [keys, rng_c, rng_w], dict_texts=[None, DICT8_TEXTS, None])
    rng_c = _with_specials([200, 128, 255], rng.integers(0, 256, m), np.uint8)
    rng_w = rng.integers(0, 1000, m)
    from oracle import oracle as O
    return mk().set_dict_hashes(O.hashbpchar), mk().set_dict_hashes(capi.hashbpchar)


def scan(relid, rel, names, quals=()):
    return P.SeqScan(relid, [(nme, P.Var(relid, *rel.var(nme))) for nme in names], quals)


def q_lt(rel, relid=1, bound=70):
    return [P.OpExpr(P.OP_LT, P.Var(relid, rel.attno("q"), P.INT4), P.Const(P.INT4, bound))]


def cols_of(rel):
    return [nme for nme in rel.names]


# ---- splitting rows into the senders' shards ----

def split(rel_pair, nsegs, how="even", seed=0):
    """per-segment range tables (oracle, product) of one relation: "even" cuts a permutation into nsegs pieces, "hole" leaves
    segment 1 empty, a list gives each segment's row count"""
    fo, fp = rel_pair
    n = fo.nrows
    perm = np.random.default_rng(seed).permutation(n)
    if how == "even":
        cuts = np.array_split(perm, nsegs)
    elif how == "hole":
        cuts = np.array_split(perm, nsegs - 1)
        cuts = cuts[:1] + [perm[:0]] + cuts[1:]
    else:
        ends = np.cumsum([0] + list(how))
        cuts = [perm[ends[i]:ends[i + 1]] for i in range(nsegs)]
    return [[fo.take(c)] for c in cuts], [[fp.take(c)] for c in cuts]


# ---- the check ----

def _cell(v):
    return ("f8", _bits(v)) if isinstance(v, float) else v


def placement(segments, rows):
    return Counter((s, tuple(_cell(v) for v in r)) for s, r in zip(segments, rows))


def _sink_lines(err, sink):
    out = []
    for line in err.splitlines():
        if line.startswith("k_probe_chain: np "):
            w = line.split()
            if int(w[w.index("sink") + 1]) == sink:
                out.append(line)
    return out


def check_kernel(expect, names, err, sink):
    """expect: "pc" (k_probe_chain ran the sink), "pf" (k_prefilter, then k_probe_chain), "generic" (k_pipeline_generic did),
    "mixed" (both: senders with and without NULL maps), "none" (nothing was launched for the sink: no rows)"""
    pcs = _sink_lines(err, sink)
    if expect in ("pc", "pf"):
        assert pcs and GEN not in names, (expect, names, err[-3000:])
        if expect == "pf":
            assert PF in names, (names, err[-3000:])
    elif expect == "generic":
        assert not pcs and GEN in names, (expect, names, err[-3000:])
    elif expect == "mixed":
        assert pcs and GEN in names, (expect, names, err[-3000:])
    else:
        assert not pcs and GEN not in names, (expect, names, err[-3000:])


def run_cluster(ctx, capfd, plan, segs_p, generic, mem_kb=0):
    dev = [to_device(ctx, s) for s in segs_p]
    cl = capi.Cluster(ctx, dev, force_generic=generic)
    for s in range(len(dev)):
        cl.E.cb_cluster_estate(cl.h, s).contents.es_operator_mem_kb = mem_kb
    capfd.readouterr()
    ctx.trace_begin()
    try:
        res = cl.run(plan)
    finally:
        names = {nme for nme, _ in ctx.trace_end()}
        cl.close()
        for d in dev:
            for r in d:
                r.free()
    return res, names, capfd.readouterr().err


def check(ctx, oracle, capfd, plan, segs_o, segs_p, expect, generic, sink=SINK_PARTITION, mem_kb=0):
    """the (segment, row) multisets of the device and the oracle agree, and the kernel `expect` ran the sink"""
    want = oracle.execute(plan, segs_o)
    got, names, err = run_cluster(ctx, capfd, plan, segs_p, generic, mem_kb)
    gp, wp = placement(got.segments, got.rows), placement(want.segments, want.rows)
    if gp != wp:
        lost, extra = wp - gp, gp - wp
        pytest.fail("placement differs: %d rows missing (e.g. %s), %d extra (e.g. %s)"
                    % (sum(lost.values()), list(lost)[:3], sum(extra.values()), list(extra)[:3]))
    check_kernel("generic" if generic and expect != "none" else expect, names, err, sink)
    return got, want


def motion_on(child, keys):
    return P.Motion(child, P.MOTIONTYPE_HASH, keys)


def scan_motion(fo, keyexprs=None, quals=True, names=None):
    names = names or cols_of(fo)
    sc = scan(1, fo, names, q_lt(fo) if quals else ())
    nk = sum(1 for nme in names if nme.startswith("k"))
    return motion_on(sc, keyexprs(sc) if keyexprs else [P.out_var(sc, i + 1) for i in range(nk)])


def kernel_for(keyname, float_payload=False, payload_nulls=False):
    return "generic" if keyname in ("float8",) or keyname in NULLABLE or float_payload or payload_nulls else "pc"


GEN_IDS = [False, True]


def _gid(g):
    return "forced_generic" if g else "chosen"


# ---- 1. key types through a filtered scan ----

@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("nsegs", [3, 8])
@pytest.mark.parametrize("keyname,expect", [(k, kernel_for(k)) for k in KEYS] + [(k, "generic") for k in NULLABLE],
                         ids=["%s-%s" % (k, kernel_for(k)) for k in KEYS] + ["%s-generic" % k for k in NULLABLE])
def test_key_types(contexts, oracle, capfd, keyname, expect, nsegs, generic):
    pair = table(20011, keyname, seed=11 + nsegs)
    segs_o, segs_p = split(pair, nsegs)
    # k_probe_chain stores at most 8 columns: the key values travel in leading columns ahead of the row's own
    nk = sum(1 for nme in pair[0].names if nme.startswith("k"))
    names = ["k%d" % i for i in range(nk)] + (["v"] if nk < 4 else [])
    got, want = check(contexts["plain"], oracle, capfd, scan_motion(pair[0], names=names), segs_o, segs_p, expect, generic)
    if keyname != "bool":                                       # two values may share a route
        assert len(set(want.segments)) == nsegs
    if keyname == "float8":
        # every row of a family on one segment: -0 with +0, every NaN with every other NaN
        for fam in ("zero", "nan"):
            segs = {s for s, r in zip(got.segments, got.rows) if _family(r[0]) == fam}
            assert len(segs) == 1, (fam, segs)


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("keyname", ["int4", "float8"], ids=["int4_plus_1-generic", "float8_times_2-generic"])
def test_expression_keys(contexts, oracle, capfd, keyname, generic):
    pair = table(20011, keyname, seed=5)
    if keyname == "int4":
        pair[0].columns[0][pair[0].columns[0] == INT32_MAX] = INT32_MAX - 1      # k + 1 stays in int4
        pair[1].columns[0][:] = pair[0].columns[0]
        expr = lambda sc: [P.OpExpr(P.OP_ADD, P.out_var(sc, 1), P.Const(P.INT4, 1))]      # noqa: E731
    else:
        expr = lambda sc: [P.OpExpr(P.OP_MUL, P.out_var(sc, 1), P.Const(P.FLOAT8, 2.0))]  # noqa: E731
    segs_o, segs_p = split(pair, 3)
    check(contexts["plain"], oracle, capfd, scan_motion(pair[0], expr), segs_o, segs_p, "generic", generic)


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
def test_float8_and_nullable_payloads(contexts, oracle, capfd, generic):
    """an int4 key with a float8 payload (NaN payloads, -0) and a nullable int8 payload: bits and NULLs arrive as sent"""
    n = 20011
    nl = (np.random.default_rng(3).random(n) < 0.3).astype(np.uint8)
    pair = table(n, "int4", seed=6, payload_nulls=nl, float_payload=True)
    segs_o, segs_p = split(pair, 5)
    got, _ = check(contexts["plain"], oracle, capfd, scan_motion(pair[0]), segs_o, segs_p, "generic", generic)
    assert any(r[pair[0].attno("v") - 1] is None for r in got.rows)


# ---- 2. segment counts and sizes ----

SEGS = [1, 2, 3, 5, 8, 64]
SIZES = [0, 1, 31, 33, 2047, 2049, 100003]


def _size_cases():
    for nsegs in SEGS:
        for n in SIZES:
            if nsegs in (3, 64) or n in (33, 100003):
                yield nsegs, n


def _size_expect(nsegs, n):
    return "none" if n == 0 or nsegs == 1 else "pc"


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("nsegs,n", list(_size_cases()),
                         ids=["%dseg-%drows-%s" % (s, n, "identity" if s == 1 else _size_expect(s, n)) for s, n in _size_cases()])
def test_segment_counts_and_sizes(contexts, oracle, capfd, nsegs, n, generic):
    pair = table(n, "mixed2", seed=n + nsegs)
    segs_o, segs_p = split(pair, nsegs)
    # one segment: every Motion is the identity, no sink runs; the rows stay where they are
    check(contexts["plain"], oracle, capfd, scan_motion(pair[0]), segs_o, segs_p, _size_expect(nsegs, n), generic and nsegs > 1 and n > 0)


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("nsegs", [3, 8])
def test_one_empty_sender(contexts, oracle, capfd, nsegs, generic):
    pair = table(20011, "int8_alias", seed=9)
    segs_o, segs_p = split(pair, nsegs, "hole")
    assert segs_o[1][0].nrows == 0
    check(contexts["plain"], oracle, capfd, scan_motion(pair[0]), segs_o, segs_p, "pc", generic)


def test_payload_null_map_on_one_sender_only(contexts, oracle, capfd):
    """segment 1 of 3 alone has a NULL map for v: its sender runs on the generic kernel, the others on k_probe_chain, and every
    receiver gets the NULLs (the receive buffer takes a NULL map when the first sender with one is copied in)"""
    n = 30000
    pair = table(n, "int4", seed=21)
    segs_o, segs_p = split(pair, 3)
    nl = (np.random.default_rng(4).random(segs_o[1][0].nrows) < 0.25).astype(np.uint8)
    vi = pair[0].attno("v") - 1
    for segs in (segs_o, segs_p):
        segs[1][0].nulls[vi] = nl
    got, _ = check(contexts["plain"], oracle, capfd, scan_motion(pair[0]), segs_o, segs_p, "mixed", False)
    passed = segs_o[1][0].columns[pair[0].attno("q") - 1] < 70
    assert sum(1 for r in got.rows if r[vi] is None) == int(nl[passed].sum())
    assert len({s for s, r in zip(got.segments, got.rows) if r[vi] is None}) == 3


# ---- 3. plan shapes feeding the Motion ----

def join_motion(fo, do, jointype, route, dup=1):
    """fact (quals q < 70) joined on k0 = dk to dim; routed by the fact's k0, k1 ("outer") or by the dim's dictionary column c
    ("build": the sink's per-code hashes come from the build relation)"""
    sf = scan(1, fo, ["k0", "k1", "q", "v"], q_lt(fo))
    sd = scan(2, do, ["dk", "c", "w"])
    h = P.Hash(sd, [P.out_var(sd, 1)])
    targets = [("k0", P.out_var(sf, 1)), ("k1", P.out_var(sf, 2)), ("v", P.out_var(sf, 4))]
    if jointype in (P.JOIN_INNER, P.JOIN_LEFT):
        targets += [("c", P.InnerVar(2, P.DICT8)), ("w", P.InnerVar(3, P.INT8))]
    j = P.HashJoin(jointype, sf, h, [P.out_var(sf, 1)], targets)
    keys = [P.out_var(j, 4)] if route == "build" else [P.out_var(j, 1), P.out_var(j, 2)]
    return motion_on(j, keys)


def _join_table(n, seed):
    """fact keys: k0 int4 over [0, 1200) (some miss the dim), k1 dict8"""
    fo, fp = table(n, "mixed2", seed)
    k0 = np.random.default_rng(seed).integers(0, 1200, n).astype(np.int32)
    fo.columns[0][:] = k0
    fp.columns[0][:] = k0
    return fo, fp


JOINS = [("inner", P.JOIN_INNER, "outer", "pc"), ("inner", P.JOIN_INNER, "build", "pc"),
         ("semi", P.JOIN_SEMI, "outer", "pc"), ("anti", P.JOIN_ANTI, "outer", "pc"),
         ("left", P.JOIN_LEFT, "outer", "generic"), ("left", P.JOIN_LEFT, "build", "generic")]


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("jt,route,expect", [j[1:] for j in JOINS], ids=["%s-by_%s-%s" % (a, r, e) for a, _, r, e in JOINS])
def test_n1_joins(contexts, oracle, capfd, jt, route, expect, generic):
    fact = _join_table(40000, 31)
    do, dp = dim(800, 32)
    segs_o, segs_p = split(fact, 3)
    segs_o, segs_p = [rt + [do] for rt in segs_o], [rt + [dp] for rt in segs_p]
    check(contexts["plain"], oracle, capfd, join_motion(fact[0], do, jt, route), segs_o, segs_p, expect, generic)


@pytest.mark.parametrize("jt", [P.JOIN_INNER, P.JOIN_SEMI], ids=["inner-pf", "semi-pf"])
def test_prefilter_then_probe_chain(contexts, oracle, capfd, jt):
    fact = _join_table(40000, 41)
    do, dp = dim(300, 42)
    segs_o, segs_p = split(fact, 3)
    check(contexts["prefilter"], oracle, capfd, join_motion(fact[0], do, jt, "outer"), [rt + [do] for rt in segs_o],
          [rt + [dp] for rt in segs_p], "pf", False)


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("mem_kb", [0, 16], ids=["one_pass-generic", "16kb_batches-generic"])
@pytest.mark.parametrize("route", ["outer", "build"])
def test_nm_join(contexts, oracle, capfd, route, mem_kb, generic):
    """N:M (every dim key three times): the pair-driven continuation feeds the sink; under 16 KB of operator memory the build
    side is split into batches and every pass appends to the same partitions"""
    fact = _join_table(30000, 51)
    do, dp = dim(2400, 52, dup=3)
    segs_o, segs_p = split(fact, 3)
    got, _ = check(contexts["plain"], oracle, capfd, join_motion(fact[0], do, P.JOIN_INNER, route), [rt + [do] for rt in segs_o],
                   [rt + [dp] for rt in segs_p], "generic", generic, mem_kb=mem_kb)
    if mem_kb:
        assert max(v["hashjoin_nbatch"] for si in got.segment_instrument for v in si.values()) >= 2


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
def test_partial_aggregate_states(contexts, oracle, capfd, generic):
    """partial HashAggregate by a nullable int4 (NULL is a group) -> hash Motion -> final aggregate on each segment: a group's
    final row exists on the segment its partial states were sent to, with every state merged"""
    n = 50000
    pair = table(n, "null_one", seed=62)
    for r in pair:
        r.columns[0][:] = r.columns[0] % 97
    segs_o, segs_p = split(pair, 3)
    sc = scan(1, pair[0], ["k0", "v", "q"])
    from cloudberry_b200.tpch import _child_var
    v = _child_var(sc)
    aggs = [("s", P.Aggref(P.AGG_SUM, v("v"))), ("n", P.Aggref(P.AGG_COUNT_STAR)), ("a", P.Aggref(P.AGG_AVG, v("q"))),
            ("mx", P.Aggref(P.AGG_MAX, v("v")))]
    partial = P.Agg(sc, P.AGG_HASHED, P.AGGSPLIT_INITIAL_SERIAL, [1], [("k0", v("k0"))] + aggs, num_groups=128)
    red = motion_on(partial, [P.out_var(partial, 1)])
    finals = [(nme, P.Aggref(ar.op, P.OuterVar(2 + i, *P.out_type(red, 2 + i)), restype=ar.restype, dscale=ar.dscale))
              for i, (nme, ar) in enumerate(aggs)]
    final = P.Agg(red, P.AGG_HASHED, P.AGGSPLIT_FINAL_DESERIAL, [1], [("k0", P.out_var(red, 1))] + finals, num_groups=128)
    got, want = check(contexts["plain"], oracle, capfd, final, segs_o, segs_p, "generic", generic)
    assert any(r[0] is None for r in want.rows) and len(want.rows) == 98


@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("nsegs", [3, 5])
def test_redistribute_of_a_redistribute(contexts, oracle, capfd, nsegs, generic):
    """the second Motion's sender drives the relation the first one delivered, and routes on other keys"""
    pair = table(30011, "mixed3", seed=71)
    segs_o, segs_p = split(pair, nsegs)
    sc = scan(1, pair[0], cols_of(pair[0]), q_lt(pair[0]))
    first = motion_on(sc, [P.out_var(sc, 1)])
    second = motion_on(first, [P.out_var(first, 2), P.out_var(first, 6)])
    check(contexts["plain"], oracle, capfd, second, segs_o, segs_p, "pc", generic)


# ---- 4. the staged pass's exact-size redo ----

@pytest.mark.parametrize("generic", GEN_IDS, ids=lambda g: "forced_generic" if g else "pc")
@pytest.mark.parametrize("skew", [True, False], ids=["skewed-redo", "uniform-no_redo"])
def test_exact_size_redo(contexts, oracle, capfd, skew, generic):
    """1.2 M rows on 3 senders, 1.1 M of them on sender 0: its first pass reserves an even share plus a quarter per destination;
    with 90 % of the rows on one key one destination overflows it and the counts of that pass size an exact second one"""
    n = 1_200_000
    rng = np.random.default_rng(81)
    k = rng.integers(INT32_MIN, INT32_MAX, n).astype(np.int32)
    if skew:
        k[rng.random(n) < 0.92] = 12345
    v = rng.integers(-10 ** 15, 10 ** 15, n)

    def mk():
        return HostRelation("fact", ["k0", "v"], [P.INT4, P.INT8], [k, v])
    segs_o, segs_p = split((mk(), mk()), 3, [1_100_000, 50_000, 50_000])
    sc = scan(1, segs_o[0][0], ["k0", "v"])
    plan = motion_on(sc, [P.out_var(sc, 1)])
    got, _ = check(contexts["plain"], oracle, capfd, plan, segs_o, segs_p, "pc", generic)
    redo = sum(si[plan.plan.plan_node_id]["motion_repartitions"] for si in got.segment_instrument)
    assert redo == (1 if skew else 0), got.segment_instrument


# ---- 5. Broadcast and Gather ----

@pytest.mark.parametrize("generic", GEN_IDS, ids=_gid)
@pytest.mark.parametrize("mtype", [P.MOTIONTYPE_BROADCAST, P.MOTIONTYPE_GATHER], ids=["broadcast-pc", "gather-pc"])
def test_broadcast_and_gather(contexts, oracle, capfd, mtype, generic):
    pair = table(20011, "dict32", seed=91)
    segs_o, segs_p = split(pair, 3)
    sc = scan(1, pair[0], cols_of(pair[0]), q_lt(pair[0]))
    got, want = check(contexts["plain"], oracle, capfd, P.Motion(sc, mtype), segs_o, segs_p, "pc", generic, sink=SINK_MATERIALIZE)
    if mtype == P.MOTIONTYPE_GATHER:
        assert set(got.segments) == {0}
    else:
        per = Counter(got.segments)
        assert set(per) == {0, 1, 2} and len(set(per.values())) == 1


# ---- 6. the direct (peer-memory) transport: one process per segment ----

@pytest.mark.parametrize("nranks", [2, 3])
def test_direct_motion_routes(nranks):
    """tests/motion_routes_worker.py under torch.distributed.run, every rank on device 0 with peer-memory windows: the rows the
    sink stored into each rank's window are the oracle's rows for that segment"""
    env = dict(os.environ, CB_BOOT="gloo", CBGPU_MOTION_WINDOW_MB="512", CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", str(nranks), "--master_port",
           str(29641 + nranks), os.path.join(root, "tests", "motion_routes_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=900, cwd=root)
    assert p.returncode == 0 and "MOTION ROUTES PASS" in p.stdout, (p.stdout[-3000:], p.stderr[-5000:])
