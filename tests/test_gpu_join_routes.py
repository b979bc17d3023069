"""Hash-join key domains through every probe route, CUDA executor vs the CPU oracle (-m gpu).

A join key reaches the build table by one of several routes, and the host picks the route from data-dependent thresholds:
k_probe_chain with the table staged in shared memory (mode 2, a few thousand slots), behind its Bloom filter in HBM
(mode 0), straight to the table after the prefilter pass applied the filter (mode 1), with probe 0 fused into the scan
stage or not (fuse0), as a chain of probes ending in SEMI / ANTI; the generic interpreter; the N:M pair probe; and, under an
operator memory budget, one pass per batch of the build side.  Tables keep single integer keys in the slot itself when they
can (int8: every build key in [0, 2^32)), else the hash value and the row id.  The key sets here are the ones where a table
could confuse two keys: int8 keys that share their low 32 bits or their hash fold, int4 at its limits, keys of mixed width.

Every case compares the oracle's rows and checks, from the CBGPU_DEBUG lines on stderr, the route it was meant to
take.  The matrix runs again with the two kept tuning switches, CBGPU_PF_SPEC and CBGPU_BLOOM_DIV (1, 4, 64)."""
import os

import numpy as np
import pytest

from cloudberry_b200 import capi
from cloudberry_b200 import plan as P
from cloudberry_b200.relation import HostRelation
from gpu_util import canon, to_device

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
GENERIC = "k_pipeline_generic"
SETTINGS = {"default": {}, "pf_spec": {"CBGPU_PF_SPEC": "1"}, "bloom1": {"CBGPU_BLOOM_DIV": "1"},
            "bloom4": {"CBGPU_BLOOM_DIV": "4"}, "bloom64": {"CBGPU_BLOOM_DIV": "64"}}
PREFILTER = {"CBGPU_PREFILTER_MIN_ROWS": "1", "CBGPU_PREFILTER_KEEP_DIV": "1"}


def _context(env):
    """a context created under `env` (knobs are read when a context is created), with the debug lines on"""
    env = dict(env, CBGPU_DEBUG="1")
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return capi.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def contexts():
    made = {}

    def get(setting, prefilter):
        if (setting, prefilter) not in made:
            made[(setting, prefilter)] = _context(dict(SETTINGS[setting], **(PREFILTER if prefilter else {})))
        return made[(setting, prefilter)]
    yield get
    for c in made.values():
        c.close()


# ---- key sets: (build key pool, probe keys, outer key types, inner key types); the pool's first keys are the special ones --

def _jh_int8(v):
    """the table's int8 key hash (jh_int8 in common.cuh): hashint8's fold, then a 32-bit mix"""
    v = int(v)
    lo, hi = v & 0xFFFFFFFF, (v >> 32) & 0xFFFFFFFF
    x = lo ^ (hi if v >= 0 else (~hi & 0xFFFFFFFF))
    x ^= x >> 16
    x = (x * 0x7feb352d) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846ca68b) & 0xFFFFFFFF
    return x ^ (x >> 16)


def _last_batch_key(start, step):
    """the first key from `start` by `step` whose hash has its top 12 bits set: it lies in the last batch of a table split
    into any power of two up to 4096 batches (the batch is the hash's top bits), so never in batch 0"""
    v = start
    while _jh_int8(v) >> 20 != 0xFFF:
        v += step
    return v


OOD_BIG = _last_batch_key(2 ** 40 + 3, 1)          # an int8 build key >= 2^32
OOD_NEG = _last_batch_key(-5, -1)                  # a negative int8 build key


def _unique(rng, lo, hi, n, avoid=()):
    out = set(int(x) for x in avoid)
    vals = []
    while len(vals) < n:
        for x in rng.integers(lo, hi, 2 * n):
            x = int(x)
            if x not in out:
                out.add(x)
                vals.append(x)
                if len(vals) == n:
                    break
    return np.array(vals, dtype=np.int64)


def _probe(rng, pool, nf, extra, miss):
    hits = rng.choice(pool, nf // 2)
    tail = np.concatenate([np.asarray(extra, dtype=np.int64), miss(nf - nf // 2 - len(extra))])
    return rng.permutation(np.concatenate([hits, tail]))


def keyset(name, npool, nf, seed):
    rng = np.random.default_rng(seed)
    u32 = lambda k: rng.integers(0, 2 ** 32, k)                        # noqa: E731
    if name in ("int8_in", "int8_big", "int8_neg", "int8_alias"):
        special = {"int8_in": [0, 1, 2 ** 32 - 1, 7], "int8_big": [OOD_BIG, 2 ** 32 - 1, 7],
                   "int8_neg": [OOD_NEG, 2 ** 32 - 1, 7], "int8_alias": [0, 2 ** 32 - 1, 7]}[name]
        pool = np.concatenate([np.array(special, dtype=np.int64), _unique(rng, 0, 2 ** 32, npool - len(special), special)])
        extra = {"int8_in": [],
                 "int8_big": [OOD_BIG, OOD_BIG & 0xFFFFFFFF, OOD_BIG + 2 ** 32],
                 "int8_neg": [OOD_NEG, OOD_NEG & 0xFFFFFFFF, OOD_NEG - 2 ** 32],
                 "int8_alias": [-1, 7 + 2 ** 32, 7 - 2 ** 32, 2 ** 32, -2 ** 32, 2 ** 33 - 1]}[name]
        if name == "int8_alias":
            some = rng.choice(pool, 2000)
            extra = extra + list(some + 2 ** 32) + list(some - 2 ** 32)
        return [pool], [_probe(rng, pool, nf, extra, u32)], [P.INT8], [P.INT8]
    if name == "int8_fold":
        # x and x ^ (m << 32 | m): the same hashint8 fold (lo ^ hi) and the same table hash; both sides hold both
        x = _unique(rng, 2 ** 32, 2 ** 40, npool // 2)
        m = rng.integers(1, 2 ** 30, npool // 2)
        pool = np.stack([x, x ^ ((m << 32) | m)], axis=1).reshape(-1)
        return [pool], [_probe(rng, pool, nf, [], lambda k: rng.integers(2 ** 32, 2 ** 40, k))], [P.INT8], [P.INT8]
    if name in ("int4", "date"):
        special = [INT32_MIN, INT32_MAX, -1, 0] if name == "int4" else [-1, 0]
        lo, hi = (INT32_MIN, INT32_MAX) if name == "int4" else (-40000, 40000)
        pool = np.concatenate([np.array(special, dtype=np.int64), _unique(rng, lo, hi, npool - len(special), special)])
        t = P.INT4 if name == "int4" else P.DATE
        return ([pool.astype(np.int32)], [_probe(rng, pool, nf, special, lambda k: rng.integers(lo, hi, k)).astype(np.int32)],
                [t], [t])
    if name == "dict8":
        pool = rng.permutation(256)[:min(npool, 200)].astype(np.uint8)
        return [pool], [rng.integers(0, 256, nf).astype(np.uint8)], [P.DICT8], [P.DICT8]
    if name == "two":
        flat = _unique(rng, 0, 100 * 2 ** 20, npool)
        pa, pb = (flat // 2 ** 20 - 50).astype(np.int32), (flat % 2 ** 20) * 4099
        idx = rng.integers(0, npool, nf)
        hit = rng.random(nf) < 0.5
        fa = np.where(hit, pa[idx], rng.integers(-50, 50, nf)).astype(np.int32)
        fb = np.where(hit, pb[idx], rng.integers(0, 2 ** 20, nf) * 4099 + rng.integers(0, 2, nf))
        return [pa, pb], [fa, fb], [P.INT4, P.INT8], [P.INT4, P.INT8]
    if name == "int4_x_int8":
        # int4 probe keys against int8 build keys, some of them outside int32 with an in-range low half
        inr = _unique(rng, INT32_MIN, INT32_MAX, npool // 2, (INT32_MIN, INT32_MAX, -1, 0))
        pool = np.concatenate([np.array([INT32_MIN, INT32_MAX, -1, 0], dtype=np.int64), inr,
                               inr[: npool - npool // 2 - 4] + 2 ** 32])
        probe = _probe(rng, inr, nf, [INT32_MIN, INT32_MAX, -1, 0], lambda k: rng.integers(INT32_MIN, INT32_MAX, k))
        return [pool], [probe.astype(np.int32)], [P.INT4], [P.INT8]
    if name == "int8_x_int4":
        # int8 probe keys, many outside int32 with the low half of a build key, against int4 build keys
        pool = np.concatenate([np.array([INT32_MIN, INT32_MAX, -1, 0], dtype=np.int64),
                               _unique(rng, INT32_MIN, INT32_MAX, npool - 4, (INT32_MIN, INT32_MAX, -1, 0))])
        some = rng.choice(pool, 3000)
        extra = list(some + 2 ** 32) + list(some - 2 ** 32) + [2 ** 31, -2 ** 31 - 1, 2 ** 32 - 1]
        return [pool.astype(np.int32)], [_probe(rng, pool, nf, extra, lambda k: rng.integers(-2 ** 40, 2 ** 40, k))], [P.INT8], [P.INT4]
    raise ValueError(name)


KEYSETS = ["int8_in", "int8_big", "int8_neg", "int8_alias", "int8_fold", "int4", "date", "dict8", "two", "int4_x_int8",
           "int8_x_int4"]


def kind(name):
    """PcProbe.kind the probe should get: 0 one int4 / date key, 1 one int8 key, 2 anything else; None: mixed widths"""
    return {"int4": 0, "date": 0, "dict8": 2, "two": 2, "int4_x_int8": None, "int8_x_int4": None}.get(name, 1)


DICT = ["v%03d" % i for i in range(256)]


def _rel(name, keys, ktypes, extra):
    n = len(keys[0])
    names = ["k%d" % i for i in range(len(keys))] + [e[0] for e in extra]
    types = list(ktypes) + [e[1] for e in extra]
    cols = list(keys) + [e[2](n) for e in extra]
    dts = [DICT if t == P.DICT8 and i < len(keys) else (["g%d" % j for j in range(5)] if names[i] == "g" else None)
           for i, t in enumerate(types)]

    def mk():
        return HostRelation(name, names, types, cols, dict_texts=dts)
    from oracle import oracle as O
    return mk().set_dict_hashes(O.hashbpchar), mk().set_dict_hashes(capi.hashbpchar)


def fact_rel(keys, ktypes, seed):
    rng = np.random.default_rng(seed)
    return _rel("fact", keys, ktypes, [("q", P.INT4, lambda n: rng.integers(0, 100, n).astype(np.int32)),
                                       ("amt", P.NUMERIC, lambda n: rng.integers(0, 10 ** 6, n)),
                                       ("g", P.DICT8, lambda n: rng.integers(0, 5, n).astype(np.uint8))])


def dim_rel(keys, ktypes, seed):
    rng = np.random.default_rng(seed)
    return _rel("dim", keys, ktypes, [("w", P.INT8, lambda n: rng.integers(0, 1000, n))])


def _scan(relid, rel, names, quals=()):
    return P.SeqScan(relid, [(nme, P.Var(relid, *rel.var(nme))) for nme in names], quals)


def join_plan(fo, dims, jointypes, qual, group_by_key=False):
    """fact joined to dims[0..] in turn (each on all its key columns against the fact's), then aggregated by g (and by the
    fact's first key column)"""
    nk = sum(1 for nme in fo.names if nme.startswith("k"))
    knames = ["k%d" % i for i in range(nk)]
    quals = [P.OpExpr(P.OP_LT, P.Var(1, fo.attno("q"), P.INT4), P.Const(P.INT4, 70))] if qual else []
    outer = _scan(1, fo, knames + ["amt", "g"], quals)
    cols = knames + ["amt", "g"]                      # the outer stream's columns, by name
    for i, (do, jt) in enumerate(zip(dims, jointypes)):
        sd = _scan(2 + i, do, knames + ["w"])
        h = P.Hash(sd, [P.out_var(sd, j + 1) for j in range(nk)])
        targets = [(c, P.out_var(outer, cols.index(c) + 1)) for c in cols]
        if jt == P.JOIN_INNER:
            targets.append(("w%d" % i, P.InnerVar(nk + 1, P.INT8)))
        outer = P.HashJoin(jt, outer, h, [P.out_var(outer, cols.index(k) + 1) for k in knames], targets)
        cols = [t[0] for t in targets]
    from cloudberry_b200.tpch import _child_var
    v = _child_var(outer)
    keys = ["g"] + (["k0"] if group_by_key else [])
    aggs = [("s", P.Aggref(P.AGG_SUM, v("amt"))), ("n", P.Aggref(P.AGG_COUNT_STAR))]
    aggs += [("sw", P.Aggref(P.AGG_SUM, v("w0")))] if "w0" in cols else []     # k_probe_chain sums at most two terms
    return P.Agg(outer, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, [cols.index(k) + 1 for k in keys], [(k, v(k)) for k in keys] + aggs,
                 num_groups=50000 if group_by_key else 64)


# route -> (build pool size, build row counts per probe, duplicate factor, join types, qual, prefilter ctx, budget, generic)
ROUTES = {
    "smem": (1500, [1500], 1, [P.JOIN_INNER], True, False, 0, False),
    "hbm_fuse0": (5000, [5000], 1, [P.JOIN_INNER], True, False, 0, False),
    "hbm": (5000, [5000], 1, [P.JOIN_INNER], False, False, 0, False),
    "prefilter": (5000, [5000], 1, [P.JOIN_INNER], True, True, 0, False),
    "chain_semi": (5000, [1000, 5000, 500], 1, [P.JOIN_INNER, P.JOIN_INNER, P.JOIN_SEMI], True, False, 0, False),
    "chain_anti": (5000, [1000, 5000, 500], 1, [P.JOIN_INNER, P.JOIN_INNER, P.JOIN_ANTI], False, False, 0, False),
    "generic": (5000, [5000], 1, [P.JOIN_INNER], True, False, 0, True),
    "nm": (1000, [1000], 3, [P.JOIN_INNER], True, False, 0, False),
    "batched_n1": (5000, [5000], 1, [P.JOIN_INNER], True, False, 16, False),
    "batched_nm": (2000, [2000], 3, [P.JOIN_INNER], True, False, 16, False),
}
SMALL_ONLY = {"smem", "generic", "nm"}      # routes a key set with only a few hundred distinct keys (dict8) can take


def _cases():
    for ks in KEYSETS:
        for route in ROUTES:
            if ks == "dict8" and route not in SMALL_ONLY:
                continue
            yield ks, route


def _chain_lines(err):
    """(modes, fuse0, np) of every k_probe_chain launch, from its two debug lines"""
    out, modes = [], None
    for line in err.splitlines():
        if line.startswith("k_probe_chain: modes "):
            w = line.split()
            modes = tuple(int(x) for x in w[2:6])
            fuse0 = int(w[-1])
        elif line.startswith("k_probe_chain: np ") and modes is not None:
            out.append((modes, fuse0, int(line.split()[2])))
            modes = None
    return out


def check_route(route, ks, err, name, nbatch, nprobes):
    joins = [c for c in _chain_lines(err) if c[2] >= 1]
    k = kind(ks)
    if route in ("generic", "batched_n1"):
        assert joins == [] and name == GENERIC, (joins, name)
        return
    if route in ("nm", "batched_nm"):
        assert "k_probe_chain: pipeline not matched (reason 1," in err, err
        return
    assert len(joins) == 1 and joins[0][2] == nprobes, joins
    modes, fuse0, _ = joins[0]
    if route == "smem":
        assert modes[0] == 2 and fuse0 == 0, joins
    elif route == "hbm_fuse0":
        assert modes[0] == 0, joins
        if k is not None:
            assert fuse0 == (1 if k in (0, 1) else 0), joins
    elif route == "hbm":
        assert modes[0] == 0 and fuse0 == 0, joins
    elif route == "prefilter":
        assert "k_prefilter: " in err, err
        if k is not None:
            assert modes[0] == (1 if k in (0, 1) else 0), joins
    elif route.startswith("chain"):
        assert modes[:3] == (2, 0, 2), joins
    assert name == "k_probe_chain"


def run_route(ctx, oracle, capfd, ks, route, seed=7):
    npool, sizes, dup, jts, qual, _pf, budget, generic = ROUTES[route]
    pool, probe, otypes, itypes = keyset(ks, npool, 20011, seed)
    fo, fp = fact_rel(probe, otypes, seed + 1)
    dims = []
    for i, nd in enumerate(sizes):
        take = np.arange(min(nd, len(pool[0])))      # every table holds the pool's special keys
        keys = [np.repeat(p[take], dup) for p in pool]
        dims.append(dim_rel(keys, itypes, seed + 2 + i))
    plan = join_plan(fo, [d[0] for d in dims], jts, qual, group_by_key=ks == "int8_fold" and route != "nm")
    want = oracle.execute(plan, [[fo] + [d[0] for d in dims]]).rows
    dev = to_device(ctx, [fp] + [d[1] for d in dims])
    for i, t in enumerate(itypes):
        if t == P.DICT8:                              # dictionary codes are compared: the sides must share one dictionary
            for d in dev[1:]:
                ctx.check(ctx.L.cbgpu_rel_share_dict_hash(d.h, i, dev[0].h, i))
    ex = capi.Executor(ctx, dev, force_generic=generic, operator_mem_kb=budget)
    capfd.readouterr()
    try:
        try:
            res = ex.run(plan)
        except capi.CbgpuError:
            if kind(ks) is None:
                return None                              # a refusal is an answer for mixed-width keys; a wrong row is not
            raise
        name = ctx.last_kernel()[0]
        batches = int(ex.estate.contents.es_hashjoin_batches_run)
    finally:
        ex.close()
        for d in dev:
            d.free()
    err = capfd.readouterr().err
    assert canon(res.rows) == canon(want), (ks, route)
    assert len(want) > 0
    nbatch = max(v["hashjoin_nbatch"] for v in res.instrument.values())
    if budget:
        assert nbatch >= 2 and batches > 0, (nbatch, batches)
    check_route(route, ks, err, name, nbatch, len(jts))
    return res.rows


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("ks,route", list(_cases()))
def test_join_route(contexts, oracle, capfd, ks, route, setting):
    run_route(contexts(setting, ROUTES[route][5]), oracle, capfd, ks, route)


@pytest.mark.parametrize("setting", ["pf_spec", "bloom1", "bloom4", "bloom64"])
def test_prefilter_pass_with_kept_switches(oracle, setting):
    """test_gpu_edge.test_prefilter_pass_on_small_inputs, in a context with CBGPU_PF_SPEC or CBGPU_BLOOM_DIV set"""
    from test_gpu_edge import test_prefilter_pass_on_small_inputs
    env = SETTINGS[setting]
    for k, v in env.items():
        os.environ[k] = v
    try:
        test_prefilter_pass_on_small_inputs(oracle)
    finally:
        for k in env:
            del os.environ[k]
