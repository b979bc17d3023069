"""HAVING as the kernel decides it (cloudberry_b200/csrc/having_eval.cuh, compiled for the host) against an independent
reference (tests/having_ref.py): exact values as fractions.Fraction, float8 values as Python floats, overflow when a
cross-product leaves the signed 128-bit range.  Random programs of compares under AND / OR / NOT over grouping columns,
constants and aggregate states, with states at +-2^127, cross-products just inside and just past 128 bits, N = 0, NaN, +-0,
+-inf and scales 0 to 18 on both sides.  Plain and under AddressSanitizer + UBSan.  Not gpu: k_having_eval runs the same
source, and tests/test_gpu_having.py holds its selections against the same reference."""
import os
import random
import shutil
import struct
import subprocess

import pytest

import having_ref as H

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "having_host.c")
CUDA_INC = "/usr/local/cuda/include"
N_CASES = 120000


def run_host(exe, cases):
    buf = [struct.pack("<i", len(cases))]
    for cols, ops, _ in cases:
        buf.append(struct.pack("<ii", len(cols), len(ops)))
        for w, vals, nulls, _f8 in cols:
            buf.append(struct.pack("<iBq", w, nulls[0], vals[0]))
        for code, a, imm in ops:
            buf.append(struct.pack("<iiq", code, a, imm))
    out = subprocess.run([exe], input=b"".join(buf), stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)
    assert len(out.stdout) == 8 * len(cases), out.stderr.decode()[-2000:]
    return struct.unpack("<%dQ" % len(cases), out.stdout)


def _build(tmp, name, extra):
    cc = shutil.which("gcc") or shutil.which("cc")
    if not cc:
        pytest.skip("no C compiler")
    exe = str(tmp / name)
    subprocess.check_call([cc, "-std=gnu11", "-O1", "-g", "-Wall", "-Werror"] + extra + ["-o", exe, SRC])
    return exe


def _check(exe, seed, n):
    rng = random.Random(seed)
    cases = [H.random_case(rng) for _ in range(n)]
    got = run_host(exe, cases)
    bad, stats = [], {"true": 0, "false": 0, "overflow": 0, "f8": 0}
    for (cols, ops, nq), r in zip(cases, got):
        bits, ovf = H.evaluate(ops, cols, 0)
        if (r & 0xFFFFFFFF, bool(r >> 32)) != (bits, ovf):
            bad.append((cols, ops, nq, hex(r), bits, ovf))
        stats["overflow"] += ovf
        stats["true" if bits == (1 << nq) - 1 else "false"] += 1
        stats["f8"] += any(op[0] >= H.CBP_FEQ and op[0] < H.CBP_FEQ + 6 for op in ops)
    assert not bad, bad[:5]
    return stats


def test_having_matches_reference(tmp_path):
    stats = _check(_build(tmp_path, "having_host", []), 20261018, N_CASES)
    # the corpus reaches every outcome
    assert stats["true"] > 10000 and stats["false"] > 10000 and stats["overflow"] > 1000 and stats["f8"] > 10000, stats


def test_having_under_sanitizers(tmp_path):
    try:
        exe = _build(tmp_path, "having_host_san", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])
    except subprocess.CalledProcessError:
        pytest.skip("the C compiler has no AddressSanitizer / UBSan runtime")
    _check(exe, 20261019, N_CASES)
