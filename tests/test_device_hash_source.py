"""The hash functions the kernels inline, as SOURCE (cloudberry_b200/csrc/common.cuh, __host__ __device__), compiled for the host
and held against the reference's own code (not gpu): hashint4 / hashint8 / hashfloat8 / hashbpchar, murmurhash32 and
jump_consistent_hash, and the compositions every sink calls - the Motion route (cdb_route: cdbhash, cdbhashreduce) and the
group hash (agg_group_hash: TupleHashTableHash_internal) - plus the checked int64 add / sub / mul of the kernels' arithmetic.
On the device the same text runs with __ddiv_rn / __dmul_rn in the jump hash (IEEE, no contraction), which
tests/test_gpu_multirank.py and the Motion tests check against the oracle's routes.  The join table's slot format (ht_slot_entry,
ht_probe_tag, ht_tag_match, ht_key_in_domain) is the same kind of source and is held against its rule over the key sets
tests/test_gpu_join_routes.py joins on."""
import ctypes as C
import os
import random
import shutil
import struct
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "..", "oracle", "_ref", "libexec_ref.so")
INT4, INT8, FLOAT8, BPCHAR, TEXT = range(5)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    so = str(tmp_path_factory.mktemp("hh") / "libhashhost.so")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "--fmad=false", "-shared",
                           "-Xcompiler", "-fPIC", "-o", so, os.path.join(HERE, "native", "hash_host.cu")])
    H = C.CDLL(so)
    for name, args in (("hh_hash_uint32", [C.c_uint32]), ("hh_hashint8", [C.c_int64]), ("hh_hashfloat8", [C.c_uint64]),
                       ("hh_hash_bpchar1", [C.c_uint8]), ("hh_hash_bytes", [C.c_char_p, C.c_int]), ("hh_murmurhash32", [C.c_uint32]),
                       ("hh_hash_combine", [C.c_uint32, C.c_uint32, C.c_int])):
        getattr(H, name).restype = C.c_uint32
        getattr(H, name).argtypes = args
    H.hh_jump_consistent_hash.restype = C.c_int32
    H.hh_jump_consistent_hash.argtypes = [C.c_uint64, C.c_int32]
    keys = [C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_uint32]
    ovf = [C.c_int64, C.c_int64, C.POINTER(C.c_int)]
    for name, res, args in (("hh_jh_int8", C.c_uint32, [C.c_int64]), ("hh_jh_mix32", C.c_uint32, [C.c_uint32]),
                            ("hh_group_key", C.c_int64, [C.c_int, C.c_int64]), ("hh_group_hash", C.c_uint32, keys),
                            ("hh_cdb_route", C.c_int32, keys + [C.c_int32]), ("hh_add_ovf", C.c_int64, ovf),
                            ("hh_sub_ovf", C.c_int64, ovf), ("hh_mul_ovf", C.c_int64, ovf),
                            ("hh_key_in_domain", C.c_int, [C.c_int32, C.c_int64]),
                            ("hh_probe_tag", C.c_uint32, [C.c_int32, C.c_uint32, C.c_int64]),
                            ("hh_slot_entry", C.c_uint64, [C.c_uint32, C.c_uint32]), ("hh_slot_empty", C.c_int, [C.c_uint64]),
                            ("hh_slot_row", C.c_uint32, [C.c_uint64]), ("hh_tag_match", C.c_int, [C.c_uint64, C.c_uint32])):
        getattr(H, name).restype = res
        getattr(H, name).argtypes = args
    return H


@pytest.fixture(scope="module")
def libs(host):
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libexec_ref.so not built (the reference source tree is not here)")
    H = host
    R = C.CDLL(REF)
    R.ref_hash_datum.restype = C.c_uint32
    R.ref_hash_datum.argtypes = [C.c_int, C.c_int64, C.c_char_p, C.c_int]
    R.ref_cdbhash_segment.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_char_p),
                                      C.POINTER(C.c_uint8), C.c_int]
    R.ref_jump_consistent_hash.argtypes = [C.c_uint32, C.c_int]
    P = C.CDLL(os.path.join(HERE, "..", "oracle", "_ref", "libpg_hashfn.so"))
    P.ref_murmurhash32.restype = C.c_uint32
    P.ref_murmurhash32.argtypes = [C.c_uint32]
    return H, R, P


def test_stored_reference_answers(host):
    """the kernels' hash source against answers of the reference's compiled hashfn.o stored in tests/test_oracle_hash.py
    (hash_uint32, bpchar, float8, and the segment of a single int4 key under cdbhash + jump_consistent_hash): runs without
    the reference tree"""
    from test_oracle_hash import KNOWN_CHAR, KNOWN_SEG3, KNOWN_SEG8, KNOWN_U32
    H = host
    for k, h in KNOWN_U32.items():
        assert H.hh_hash_uint32(k) == h
    for ch, h in KNOWN_CHAR.items():
        assert H.hh_hash_bpchar1(ord(ch)) == h
    assert H.hh_hashfloat8(_bits(1.5)) == 0x259a2972 and H.hh_hashfloat8(_bits(-0.0)) == 0
    for known, nseg in ((KNOWN_SEG8, 8), (KNOWN_SEG3, 3)):
        for k, seg in known.items():
            assert H.hh_jump_consistent_hash(H.hh_hash_combine(0, H.hh_hash_uint32(k), 0), nseg) == seg
            for t in (CB_INT4, CB_DATE):
                assert _call_keys(H.hh_cdb_route, [t], [k - (1 << 32) if k >= (1 << 31) else k], [0], None, nseg) == seg


def _bits(f):
    return struct.unpack("<Q", struct.pack("<d", f))[0]


def _s64(u):
    return u - (1 << 64) if u >= (1 << 63) else u


# CbTypeId (include/cb_plan.h) of the kernels' key types
CB_INT4, CB_INT8, CB_DATE, CB_BPCHAR1, CB_DICT32, CB_FLOAT8 = 1, 2, 3, 5, 7, 8
REF_KIND = {CB_INT4: INT4, CB_DATE: INT4, CB_INT8: INT8, CB_FLOAT8: FLOAT8, CB_BPCHAR1: BPCHAR, CB_DICT32: BPCHAR}
WORDS = ["", "A", "ASIA", "MACHINERY", "1-URGENT", "a longer string than twelve bytes", "Brand#13 ", "\u00e9t\u00e9"]


def _call_keys(fn, types, vals, nulls, dicts, *extra):
    """fn(nkeys, types, dicts, keys, knull, *extra) over ctypes arrays; dicts[k] is a list of per-code hashes or None"""
    n = len(types)
    tables = [(C.c_uint32 * len(d))(*d) if d else None for d in (dicts or [None] * n)]
    ptrs = (C.c_void_p * n)(*[C.cast(t, C.c_void_p) if t is not None else None for t in tables])
    knull = sum(1 << k for k, nul in enumerate(nulls) if nul)
    return fn(n, (C.c_int32 * n)(*types), ptrs, (C.c_int64 * n)(*vals), knull, *extra)


def _random_keys(rng, R):
    """1-4 keys of the kernels' key types with NULLs; per key: type, device value, the reference's (bits, string), dictionary"""
    word_hash = [R.ref_hash_datum(BPCHAR, 0, w.encode(), len(w.encode())) for w in WORDS]
    keys = []
    for _ in range(rng.randrange(1, 5)):
        t = rng.choice([CB_INT4, CB_DATE, CB_INT8, CB_FLOAT8, CB_BPCHAR1, CB_DICT32])
        d, s = None, None
        if t in (CB_INT4, CB_DATE):
            v = rng.choice([0, -1, -2 ** 31, 2 ** 31 - 1, rng.getrandbits(32) - 2 ** 31])
        elif t == CB_INT8:
            v = rng.choice([0, -1, -2 ** 63, 2 ** 63 - 1, rng.getrandbits(64) - 2 ** 63])
        elif t == CB_FLOAT8:
            v = _s64(rng.choice([_bits(0.0), _bits(-0.0), 0x7ff8000000000000, 0xfff0000000000001, 0x7ff0000000000123,
                                 _bits(float("inf")), _bits(rng.uniform(-1e9, 1e9))]))
        elif t == CB_BPCHAR1:
            v = rng.randrange(1, 256)
            s = bytes([v])
        else:
            v = rng.randrange(len(WORDS))
            d, s = word_hash, WORDS[v].encode()
        keys.append((t, v, s, d, 1 if rng.random() < 0.15 else 0))
    return keys


def test_type_hash_functions(libs):
    H, R, _ = libs
    rng = random.Random(77)
    for k in [0, 1, 42, 0x7fffffff, 0x80000000, 0xffffffff] + [rng.getrandbits(32) for _ in range(5000)]:
        s = k - (1 << 32) if k >= (1 << 31) else k
        assert H.hh_hash_uint32(k) == R.ref_hash_datum(INT4, s, None, 0)
    for v in [0, 1, -1, 2 ** 31, -2 ** 31 - 1, 2 ** 63 - 1, -2 ** 63] + [rng.getrandbits(64) - 2 ** 63 for _ in range(5000)]:
        assert H.hh_hashint8(v) == R.ref_hash_datum(INT8, v, None, 0), v
    fl = [0.0, -0.0, 1.5, float("inf"), float("-inf"), float("nan"), 5e-324, 1.7e308] + [rng.uniform(-1e15, 1e15) for _ in range(3000)]
    for f in fl:
        assert H.hh_hashfloat8(_bits(f)) == R.ref_hash_datum(FLOAT8, _s64(_bits(f)), None, 0), f
    for nan_bits in (0xfff8000000000001, 0x7ff0000000000001, 0xffffffffffffffff):
        assert H.hh_hashfloat8(nan_bits) == R.ref_hash_datum(FLOAT8, _s64(nan_bits), None, 0)
    for ch in range(1, 256):
        assert H.hh_hash_bpchar1(ch) == R.ref_hash_datum(BPCHAR, 0, bytes([ch]), 1), ch
    for n in list(range(0, 40)) + [63, 64, 65, 500]:
        s = bytes(rng.randrange(33, 127) for _ in range(n))
        assert H.hh_hash_bytes(s, n) == R.ref_hash_datum(TEXT, 0, s, n)


def test_murmur_and_key_combination(libs):
    H, R, P = libs
    rng = random.Random(78)
    for _ in range(5000):
        x = rng.getrandbits(32)
        assert H.hh_murmurhash32(x) == P.ref_murmurhash32(x)
        nseg = rng.choice([1, 2, 3, 8, 48, 64, 1000])
        assert H.hh_jump_consistent_hash(x, nseg) == R.ref_jump_consistent_hash(x, nseg)
    # the Motion's route as the kernels compile it (cdb_route: cdbhash over the keys, then cdbhashreduce) against the
    # reference's own evalHashKey on the same keys: int4, date, int8, float8 (signed zeros and NaN payloads), bpchar(1),
    # dictionary codes whose per-code table holds hashbpchar of each string, NULLs, 1-64 segments and a few more
    for i in range(6000):
        nseg = 1 + i % 64 if i < 5000 else rng.choice([65, 100, 1000, 4096])
        keys = _random_keys(rng, R)
        ts, vs, ss, ds, ns = zip(*keys)
        nk = len(keys)
        strs = (C.c_char_p * nk)(*ss)
        want = R.ref_cdbhash_segment(nk, (C.c_int * nk)(*[REF_KIND[t] for t in ts]), (C.c_int64 * nk)(*vs), strs,
                                     (C.c_uint8 * nk)(*ns), nseg)
        assert want >= 0
        assert _call_keys(H.hh_cdb_route, ts, vs, ns, ds, nseg) == want, (keys, nseg)


def test_group_hash(libs, host):
    """agg_group_hash against TupleHashTableHash_internal composed of the reference's pieces: its hash functions, the
    rotate-xor with NULLs contributing nothing, then libpg_hashfn's murmurhash32"""
    H, R, P = libs
    rng = random.Random(80)
    for _ in range(4000):
        keys = _random_keys(rng, R)
        want = 0
        for t, v, s, d, nul in keys:
            want = ((want << 1) | (want >> 31)) & 0xffffffff
            if not nul:
                want ^= R.ref_hash_datum(REF_KIND[t], v, s, len(s) if s else 0)
        ts, vs, _, ds, ns = zip(*keys)
        assert _call_keys(H.hh_group_hash, ts, vs, ns, ds) == P.ref_murmurhash32(want), keys


def test_group_key_float8(host):
    """float8eq's groups: -0.0 and +0.0 are one key, every NaN payload is one key, and they hash alike (with a second key)"""
    H = host
    for same in ([_bits(0.0), _bits(-0.0)], [0x7ff8000000000000, 0xfff8000000000000, 0x7ff0000000000001, 0xffffffffffffffff]):
        ks = {H.hh_group_key(CB_FLOAT8, _s64(b)) for b in same}
        assert len(ks) == 1
        hs = {_call_keys(H.hh_group_hash, [CB_FLOAT8, CB_INT4], [_s64(b), 7], [0, 0], None) for b in same}
        assert len(hs) == 1
    for b in (_bits(1.5), _bits(float("inf")), _bits(float("-inf")), 1):
        assert H.hh_group_key(CB_FLOAT8, _s64(b)) == _s64(b)
    assert H.hh_group_key(CB_INT8, _s64(_bits(-0.0))) == _s64(_bits(-0.0))


def test_checked_int64_arithmetic(host):
    """i64_add_ovf / i64_sub_ovf / i64_mul_ovf: the wrapped result and whether the exact one leaves int64 (int8pl / int8mi /
    int8mul's "bigint out of range")"""
    H = host
    rng = random.Random(81)
    edges = [0, 1, 2 ** 31, 2 ** 32, 2 ** 62]
    vals = sorted({s * e for e in edges for s in (1, -1)} | {-2 ** 63, 2 ** 63 - 1, 2 ** 63 - 2, -2 ** 63 + 1, 3037000499,
                                                             3037000500})
    vals += [rng.getrandbits(64) - 2 ** 63 for _ in range(60)] + [rng.getrandbits(33) - 2 ** 32 for _ in range(30)]
    for x in vals:
        for y in vals:
            for fn, exact in ((H.hh_add_ovf, x + y), (H.hh_sub_ovf, x - y), (H.hh_mul_ovf, x * y)):
                o = C.c_int(-1)
                r = fn(x, y, C.byref(o))
                assert r == _s64(exact & (2 ** 64 - 1)), (fn.__name__, x, y)
                assert o.value == (not -2 ** 63 <= exact < 2 ** 63), (fn.__name__, x, y)


def test_join_slot_format(host):
    """a slot's tag and row round-trip, a probe's tag matches the tag its key was built with, and a key-in-slot table (keyslot 1:
    int32 domain, 2: [0, 2^32)) never confuses two keys: inside its domain distinct keys have distinct tags, and a key outside
    it is refused.  Key sets of tests/test_gpu_join_routes.py: int8 keys that share their low 32 bits or their hash fold, int4
    at its limits, int8 keys just outside [0, 2^32)."""
    H = host
    i32min, i32max = -2 ** 31, 2 ** 31 - 1
    rng = random.Random(79)
    int8_keys = [0, 1, 7, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7, 7 - 2 ** 32, -1, -2 ** 32, 2 ** 33 - 1, 2 ** 40 + 3, -5,
                 i32min, i32max] + [rng.getrandbits(32) for _ in range(2000)] + [rng.getrandbits(40) for _ in range(500)]
    int8_keys += [k + 2 ** 32 for k in int8_keys[:200]] + [k - 2 ** 32 for k in int8_keys[:200]]
    fold = {}
    for k in int8_keys:                                  # keys whose hashint8 fold (lo ^ hi, or lo ^ ~hi) agrees
        lo, hi = k & 0xFFFFFFFF, (k >> 32) & 0xFFFFFFFF
        fold.setdefault(lo ^ (hi if k >= 0 else ~hi & 0xFFFFFFFF), []).append(k)
    assert any(len(set(v)) > 1 for v in fold.values())
    int4_keys = [i32min, i32max, i32min + 1, i32max - 1, -1, 0, 1] + [rng.getrandbits(32) - 2 ** 31 for _ in range(2000)]
    assert H.hh_slot_empty(0xFFFFFFFFFFFFFFFF) and not H.hh_slot_empty(0)
    for keyslot, keys in ((2, int8_keys), (1, int4_keys), (1, int8_keys)):
        tags = {}
        for row, k in enumerate(set(keys)):
            h = H.hh_jh_int8(k) if keys is int8_keys else H.hh_jh_mix32(k & 0xFFFFFFFF)
            inside = H.hh_key_in_domain(keyslot, k)
            assert inside == ((i32min <= k <= i32max) if keyslot == 1 else (0 <= k < 2 ** 32)), (keyslot, k)
            for ks in (keyslot, 0):
                tag = H.hh_probe_tag(ks, h, k)
                e = H.hh_slot_entry(tag, row)
                assert not H.hh_slot_empty(e) and H.hh_slot_row(e) == row and H.hh_tag_match(e, tag)
                assert tag == (h if ks == 0 else k & 0xFFFFFFFF)
            if inside:
                tag = H.hh_probe_tag(keyslot, h, k)
                assert tags.setdefault(tag, k) == k, (keyslot, k, tags[tag])
