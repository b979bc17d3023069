"""Relations, plans and a numpy group-by for the tests of GROUP BY over five to eight columns (tests/test_gpu_wide_groups.py,
tests/host_wide_groups_worker.py).  Not a test by itself.

fact(fk, int4, int8, date, bpchar1, dict8, dict32, numeric, float8, v) joins dim(d_key, d_x) on fk = d_key, then groups by the
first nkeys of KEYS (or of CHAIN_KEYS) with sum(v) and count(*); scan_plan groups fact alone.  Every key column takes two or
three values, so the groups share rows; float8 takes -0, +0, two NaN bit patterns and ordinary values (float8eq puts -0 with +0 and every NaN together).
With nulls=True every key column but fk also holds NULLs, which group together."""
import math
import struct

import numpy as np

from cloudberry_b200 import plan as P
from cloudberry_b200 import tpch_q10_q18
from cloudberry_b200.relation import HostRelation

FACT = [("fk", P.INT4), ("k_int4", P.INT4), ("k_int8", P.INT8), ("k_date", P.DATE), ("k_char", P.BPCHAR1),
        ("k_dict8", P.DICT8), ("k_dict32", P.DICT32), ("k_num", P.NUMERIC), ("k_f8", P.FLOAT8), ("v", P.NUMERIC)]
DIM = [("d_key", P.INT4), ("d_x", P.INT4)]
# group keys in order: every type, float8 last (the generic interpreter takes it; the compiled probe chain does not)
KEYS = ["k_int4", "k_int8", "k_date", "k_char", "k_dict8", "k_dict32", "k_num", "k_f8", "d_x"]
# keys the probe chain's AGG sink reads straight from columns: no float8, no NULLs, one from the build side
CHAIN_KEYS = ["k_int4", "k_int8", "k_date", "k_char", "k_dict8", "k_dict32", "k_num", "d_x", "fk"]
DICT8_TEXTS = ["red", "green", "blue"]
DICT32_TEXTS = ["alpha", "beta", "gamma", "delta"]
NDIM = 50
_NAN2 = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000123))[0]
F8_VALUES = np.array([-0.0, 0.0, float("nan"), _NAN2, 1.5, -2.25], dtype=np.float64)


def tables(n, hashfn, nulls=False, seed=7):
    rng = np.random.default_rng(seed)
    cols = {
        "fk": rng.integers(0, NDIM, n).astype(np.int32),
        "k_int4": rng.integers(-1, 2, n).astype(np.int32),
        "k_int8": (rng.integers(0, 3, n) * 10**12).astype(np.int64),
        "k_date": (8000 + rng.integers(0, 3, n)).astype(np.int32),
        "k_char": np.array([ord(c) for c in "AB"], dtype=np.uint8)[rng.integers(0, 2, n)],
        "k_dict8": rng.integers(0, len(DICT8_TEXTS), n).astype(np.uint8),
        "k_dict32": rng.integers(0, len(DICT32_TEXTS), n).astype(np.int32),
        "k_num": rng.integers(-1, 2, n).astype(np.int64) * 12345,
        "k_f8": F8_VALUES[rng.integers(0, len(F8_VALUES), n)],
        "v": rng.integers(-10000, 10000, n).astype(np.int64),
    }
    nl = [None] * len(FACT)
    if nulls:
        nl = [None] + [(rng.random(n) < 0.1).astype(np.uint8) for _ in FACT[1:-1]] + [None]
    texts = [None] * len(FACT)
    texts[5], texts[6] = DICT8_TEXTS, DICT32_TEXTS
    fact = HostRelation("fact", [c for c, _ in FACT], [t for _, t in FACT], [cols[c] for c, _ in FACT], nulls=nl,
                        dict_texts=texts).set_dict_hashes(hashfn)
    dim = HostRelation("dim", [c for c, _ in DIM], [t for _, t in DIM],
                       [np.arange(NDIM, dtype=np.int32), (np.arange(NDIM) % 3).astype(np.int32)])
    return [fact, dim]


def plan(keys):
    """Agg (group by keys; sum(v), count(*)) <- Hash Join (fk = d_key) <- Seq Scan fact, Hash <- Seq Scan dim"""
    fnames = [c for c, _ in FACT]
    scan = P.SeqScan(1, [(c, P.Var(1, k + 1, t, 2 if t == P.NUMERIC else 0)) for k, (c, t) in enumerate(FACT)])
    dim = P.SeqScan(2, [(c, P.Var(2, k + 1, t)) for k, (c, t) in enumerate(DIM)])
    targets = [(c, P.out_var(scan, fnames.index(c) + 1)) for c in fnames] + [("d_x", P.InnerVar(2, P.INT4))]
    j = P.HashJoin(P.JOIN_INNER, scan, P.Hash(dim, [P.out_var(dim, 1)]), [P.out_var(scan, 1)], targets)
    names = fnames + ["d_x"]
    idx = [names.index(k) + 1 for k in keys]
    return P.Agg(j, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, idx,
                 [(k, P.out_var(j, i)) for k, i in zip(keys, idx)] +
                 [("s", P.Aggref(P.AGG_SUM, P.out_var(j, names.index("v") + 1))), ("n", P.Aggref(P.AGG_COUNT_STAR))],
                 num_groups=1000)


def scan_plan(keys):
    """Agg (group by keys; sum(v), count(*)) <- Seq Scan fact: no join, so the groups come back through the top-level
    aggregate's own read-back"""
    fnames = [c for c, _ in FACT]
    scan = P.SeqScan(1, [(c, P.Var(1, k + 1, t, 2 if t == P.NUMERIC else 0)) for k, (c, t) in enumerate(FACT)])
    idx = [fnames.index(k) + 1 for k in keys]
    return P.Agg(scan, P.AGG_HASHED, P.AGGSPLIT_SIMPLE, idx,
                 [(k, P.out_var(scan, i)) for k, i in zip(keys, idx)] +
                 [("s", P.Aggref(P.AGG_SUM, P.out_var(scan, fnames.index("v") + 1))), ("n", P.Aggref(P.AGG_COUNT_STAR))],
                 num_groups=100)


def canon_value(x):
    """one output value in a form that compares as float8eq groups: every NaN alike, -0 as +0"""
    if isinstance(x, float):
        return "NaN" if math.isnan(x) else x + 0.0
    return x


def canon(rows):
    return sorted([tuple(canon_value(v) for v in r) for r in rows], key=lambda r: tuple(map(str, r)))


def numpy_groups(fact, keys):
    """the plan's rows, grouped in Python over the host columns (no code shared with the executor)"""
    dim_x = np.arange(NDIM) % 3
    names = fact.names
    cols = {}
    for k in keys:
        if k == "d_x":
            cols[k] = [int(x) for x in dim_x[fact.columns[0]]]
            continue
        i = names.index(k)
        c, nl, t = fact.columns[i], fact.nulls[i], fact.types[i]
        vals = [tpch_q10_q18.numeric_text(x, 2) if t == P.NUMERIC else canon_value(float(x)) if t == P.FLOAT8 else int(x)
                for x in c.tolist()]
        cols[k] = [None if (nl is not None and nl[r]) else v for r, v in enumerate(vals)]
    v = fact.columns[names.index("v")]
    groups = {}
    for r in range(fact.nrows):
        g = tuple(cols[k][r] for k in keys)
        s, n = groups.get(g, (0, 0))
        groups[g] = (s + int(v[r]), n + 1)
    return canon([g + (tpch_q10_q18.numeric_text(s, 2), n) for g, (s, n) in groups.items()])
