"""Reference of HAVING over a groups relation (cbgpu_having_select, cloudberry_b200/csrc/having_eval.cuh) and a generator of
random programs, shared by tests/test_having_host.py and tests/test_gpu_having.py.  Not a test by itself.

A column is (width, values, nulls, f8): width 1 / 4 / 8 bytes, values as Python ints (float8 columns: their bit patterns),
nulls a list of 0 / 1 or None, f8 whether the column is float8.  An exact value is a fractions.Fraction, a float8 value a
Python float; NULL is None.  A compare of two non-NULL exact values overflows when either cross-product
num_a * den_b * 10^(scale_b - scale_a) (and its mirror) lies outside the signed 128-bit range - independent of the order in
which the kernel multiplies."""
import math
import struct
from fractions import Fraction

from cloudberry_b200.capi import (CBH_AVG, CBH_CONST_F8, CBH_CONST_NULL, CBH_COUNT, CBH_FAVG, CBH_FMAX, CBH_FMIN, CBH_FSUM,
                                  CBH_MAX, CBH_MIN, CBH_SUM, CBP_AND, CBP_CONST, CBP_EQ, CBP_FEQ, CBP_LOAD, CBP_NOT, CBP_OR,
                                  CBP_STATE)

I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1
F8_KINDS = (CBH_FSUM, CBH_FAVG, CBH_FMIN, CBH_FMAX)


def f8_bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def bits_f8(b):
    return struct.unpack("<d", struct.pack("<q", b))[0]


def f8ord(b):
    """CBP_F8ORD: float8 bits -> an int64 whose order is float8_cmp_internal's"""
    if math.isnan(bits_f8(b)):
        b = 0x7FF8000000000000
    return b if b >= 0 else b ^ 0x7FFFFFFFFFFFFFFF


def _signed(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def leaf(op, cols, g):
    """('x', num, den, scale) / ('f', float) / None (NULL)"""
    code, a, imm = op
    if code == CBP_LOAD:
        w, vals, nulls, f8 = cols[a]
        if nulls is not None and nulls[g]:
            return None
        return ("f", bits_f8(int(vals[g]))) if f8 else ("x", int(vals[g]), 1, imm)
    if code == CBP_CONST:
        if a & CBH_CONST_NULL:
            return None
        if a & CBH_CONST_F8:
            return ("f", bits_f8(imm))
        return ("x", imm, 1, a & 0xFFFF)
    kind, scale = imm & 0xFF, imm >> 8
    n, lo, hi = (_signed(int(cols[a + i][1][g]), 64) for i in range(3))
    if kind == CBH_COUNT:
        return ("x", n, 1, 0)
    if n == 0:
        return None
    if kind in (CBH_SUM, CBH_AVG):
        return ("x", (hi << 64) | (lo & ((1 << 64) - 1)), n if kind == CBH_AVG else 1, scale)
    if kind in (CBH_MIN, CBH_MAX):
        return ("x", lo, 1, scale)
    if kind == CBH_FSUM:
        return ("f", bits_f8(lo))
    if kind == CBH_FAVG:
        return ("f", bits_f8(lo) / n)
    return ("f", bits_f8(lo if lo >= 0 else lo ^ 0x7FFFFFFFFFFFFFFF))     # F8ORD's inverse (no NaN image is negative)


def _cmp(x, y):
    if x[0] == "f":
        a, b = x[1], y[1]
        if math.isnan(a):
            return 0 if math.isnan(b) else 1
        if math.isnan(b):
            return -1
        return (a > b) - (a < b)
    _, na, da, sa = x
    _, nb, db, sb = y
    L, R = na * db * 10 ** max(0, sb - sa), nb * da * 10 ** max(0, sa - sb)
    if not (I128_MIN <= L <= I128_MAX and I128_MIN <= R <= I128_MAX):
        return "overflow"
    fa, fb = Fraction(na, da * 10 ** sa), Fraction(nb, db * 10 ** sb)
    return (fa > fb) - (fa < fb)


def evaluate(ops, cols, g):
    """(verdict bits, overflow) of the program for group g: bit q = boolean q is true"""
    st, ovf = [], False
    for i, (code, a, imm) in enumerate(ops):
        if code in (CBP_LOAD, CBP_CONST, CBP_STATE):
            continue
        if CBP_EQ <= code < CBP_FEQ + 6:
            x, y = leaf(ops[i - 2], cols, g), leaf(ops[i - 1], cols, g)
            if x is None or y is None:
                st.append(None)
                continue
            c = _cmp(x, y)
            if c == "overflow":
                ovf, c = True, 0
            rel = (code - CBP_EQ) % 6
            st.append([c == 0, c != 0, c < 0, c <= 0, c > 0, c >= 0][rel])
        elif code in (CBP_AND, CBP_OR):
            y, x = st.pop(), st.pop()
            if code == CBP_AND:
                st.append(False if x is False or y is False else None if x is None or y is None else True)
            else:
                st.append(True if x is True or y is True else None if x is None or y is None else False)
        elif code == CBP_NOT:
            st[-1] = None if st[-1] is None else not st[-1]
    return sum(1 << q for q, v in enumerate(st) if v is True), ovf


def keep(ops, cols, g, nquals):
    bits, ovf = evaluate(ops, cols, g)
    return bits == (1 << nquals) - 1, ovf


# ---- random programs ----
SPECIAL_F8 = [0.0, -0.0, float("inf"), -float("inf"), float("nan"), 1.0, -1.0, 0.5, 1e-300, 5e-324, 1.7976931348623157e308]


def rand_f8(rng):
    r = rng.random()
    if r < 0.3:
        return rng.choice(SPECIAL_F8)
    if r < 0.6:
        return float(rng.randint(-20, 20)) / 4
    return rng.uniform(-1e6, 1e6)


def rand_i128(rng):
    r = rng.random()
    if r < 0.15:
        return rng.choice([I128_MIN, I128_MAX, I128_MIN + 1, I128_MAX - 1, 0, 1, -1])
    if r < 0.5:
        return rng.randint(-1000, 1000)
    return rng.randint(-(1 << rng.randint(1, 127)), 1 << rng.randint(1, 127))


def boundary_num(rng, mult):
    """a numerator whose product with mult lies just inside or just outside the signed 128-bit range"""
    q = (I128_MAX // mult) if rng.random() < 0.5 else -(-I128_MIN // mult)
    return max(I128_MIN, min(I128_MAX, q + rng.choice([-1, 0, 1])))


def split128(v):
    """a 128-bit value as its (lo, hi) int8 columns"""
    return _signed(v, 64), _signed(v >> 64, 64)


class Builder:
    """one random program over freshly made one-group columns (the host test) - every leaf gets its own column(s)"""

    def __init__(self, rng):
        self.rng, self.cols, self.ops = rng, [], []

    def col(self, w, v, null=0, f8=False):
        self.cols.append((w, [v], [null], f8))
        return len(self.cols) - 1

    def state(self, kind, scale, n, lo, hi=None):
        a = len(self.cols)
        lo, hi2 = split128(lo) if hi is None else (lo, hi)
        for v in (n, lo, hi2):
            self.col(8, v)
        self.ops.append((CBP_STATE, a, kind | scale << 8))

    def leaf(self, f8):
        rng = self.rng
        r = rng.random()
        scale = rng.randint(0, 18)
        if r < 0.25:
            if f8:
                self.ops.append((CBP_LOAD, self.col(8, f8_bits(rand_f8(rng)), rng.random() < 0.1, True), 0))
            else:
                w = rng.choice([1, 4, 8])
                v = rng.randint(0, 255) if w == 1 else rng.randint(-2**31, 2**31 - 1) if w == 4 else \
                    rng.choice([rng.randint(-2**63, 2**63 - 1), rng.randint(-10**6, 10**6)])
                self.ops.append((CBP_LOAD, self.col(w, v, rng.random() < 0.1), 0 if w == 1 else scale))
        elif r < 0.5:
            null = CBH_CONST_NULL if rng.random() < 0.05 else 0
            if f8:
                self.ops.append((CBP_CONST, CBH_CONST_F8 | null, f8_bits(rand_f8(rng))))
            else:
                v = rng.choice([rng.randint(-2**63, 2**63 - 1), rng.randint(-10**6, 10**6), 0, -2**63, 2**63 - 1])
                self.ops.append((CBP_CONST, scale | null, v))
        else:
            n = 0 if rng.random() < 0.1 else rng.choice([1, 2, 3, 7, rng.randint(1, 2**40), 2**63 - 1])
            if f8:
                kind = rng.choice(F8_KINDS)
                b = f8_bits(rand_f8(rng))
                self.state(kind, 0, n, f8ord(b) if kind in (CBH_FMIN, CBH_FMAX) else b, 0)
            else:
                kind = rng.choice([CBH_COUNT, CBH_SUM, CBH_AVG, CBH_MIN, CBH_MAX])
                if kind in (CBH_SUM, CBH_AVG):
                    self.state(kind, scale, n, rand_i128(rng))
                else:
                    self.state(kind, 0 if kind == CBH_COUNT else scale, n, rng.randint(-2**63, 2**63 - 1), 0)

    def boundary(self):
        """exact operands whose cross-product lies just inside or just outside 128 bits, in either order"""
        rng = self.rng
        sx = rng.randint(0, 18)
        sy = sx + rng.randint(0, 18)
        ny = rng.choice([1, 3, 7, 10**9 + 7, 2**62])
        self.state(rng.choice([CBH_SUM, CBH_AVG]), sx, 1, boundary_num(rng, ny * 10 ** (sy - sx)))
        self.state(CBH_AVG, sy, ny, rng.randint(-5, 5))
        if rng.random() < 0.5:
            self.ops[-2], self.ops[-1] = self.ops[-1], self.ops[-2]
        self.ops.append((rng.randint(CBP_EQ, CBP_EQ + 5), 0, 0))

    def compare(self):
        if self.rng.random() < 0.15:
            return self.boundary()
        f8 = self.rng.random() < 0.35
        self.leaf(f8)
        self.leaf(f8)
        self.ops.append(((CBP_FEQ if f8 else CBP_EQ) + self.rng.randint(0, 5), 0, 0))

    def boolean(self, depth):
        r = self.rng.random()
        if depth == 0 or r < 0.5:
            self.compare()
        elif r < 0.65:
            self.boolean(depth - 1)
            self.ops.append((CBP_NOT, 0, 0))
        else:
            op = CBP_AND if self.rng.random() < 0.5 else CBP_OR
            for i in range(self.rng.randint(2, 3)):
                self.boolean(depth - 1)
                if i:
                    self.ops.append((op, 0, 0))


def random_case(rng):
    """(cols, ops, nquals) over one group, at most 64 columns"""
    while True:
        b = Builder(rng)
        nq = rng.randint(1, 3)
        for _ in range(nq):
            b.boolean(2)
        if len(b.cols) <= 64:
            return b.cols, b.ops, nq
