"""The host loop of the device top-N (cbgpu_topn, ORDER BY ... LIMIT n with n <= 64) without a GPU (not gpu): libcbgpu.so over
tests/native/fake_cudart.c, a CUDA runtime that computes nothing (LD_PRELOADed into a subprocess, as
test_host_logic_fake_runtime.py does).  Every key reads back as constant there, so the threshold selection gives up on each key
and every call goes to the tournament, the host loop of k_topn passes.  Every LIMIT from 1 to 64 must return, over 4097, 10 000
and 10^6 rows, with a number of launches logarithmic in the rows: a pass that does not shrink its input would loop forever.
The refusals (key count, LIMIT range, bad key column, nullable and float8 keys) come with their code and message and before any
launch; an empty relation gives no rows."""
import json
import math
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="needs the CUDA headers")

INVALID, UNSUPPORTED = -2, -3


@pytest.fixture(scope="module")
def fake(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakecuda")
    so = str(d / "libfakecudart.so")
    subprocess.check_call(["gcc", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
                           os.path.join(ROOT, "tests", "native", "fake_cudart.c")])
    return so


def _run(so, *args, timeout=60):
    """the worker's records; a worker that does not finish fails the test with the last call that returned"""
    cmd = [sys.executable, os.path.join(ROOT, "tests", "host_topn_worker.py")] + [str(a) for a in args]
    env = dict(os.environ, LD_PRELOAD=so)
    try:
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    except subprocess.TimeoutExpired as e:
        out = e.stdout.decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
        done = [ln for ln in out.splitlines() if ln.startswith("TOPN ")]
        pytest.fail("cbgpu_topn did not return within %ds (%s); last call that returned: %s"
                    % (timeout, " ".join(map(str, args)), done[-1] if done else "none"))
    recs = [json.loads(ln[len("TOPN "):]) for ln in p.stdout.splitlines() if ln.startswith("TOPN ")]
    assert p.returncode == 0 and recs, (p.stdout[-2000:], p.stderr[-4000:])
    return recs


@pytest.mark.parametrize("n", [4097, 10000, 10**6])
def test_every_limit_returns_in_logarithmic_launches(fake, n):
    recs = _run(fake, "calls", n)
    assert [(r["nkeys"], r["limit"]) for r in recs] == [(k, lim) for k in (1, 4) for lim in range(1, 65)]
    for r in recs:
        assert r["rc"] == 0, r
        # the no-op runtime reads back zeroed indices: row 0, a row all the same, so every slot is filled
        assert r["nout"] == r["limit"], r
        # per key one k_topn_min + k_topn_kth (every key is constant here), then tournament passes that at least halve the input
        assert 0 < r["launches"] <= math.ceil(math.log2(n)) + 2 * r["nkeys"] + 2, r


def test_refusals_come_before_any_launch(fake):
    recs = {r["name"]: r for r in _run(fake, "refusals")}
    want = {"nkeys_0": (UNSUPPORTED, "1..4 sort keys and LIMIT <= 64"), "nkeys_5": (UNSUPPORTED, "1..4 sort keys and LIMIT <= 64"),
            "limit_0": (UNSUPPORTED, "got 0"), "limit_65": (UNSUPPORTED, "got 65"),
            "key_col_3": (INVALID, "bad key column 3"), "key_col_neg": (INVALID, "bad key column -1"),
            "float8_key": (UNSUPPORTED, "float8 key"), "nullable_key": (UNSUPPORTED, "nullable sort key")}
    for name, (code, frag) in want.items():
        r = recs[name]
        assert r["rc"] == code and frag in r["msg"] and r["launches"] == 0, r
    for name in ("empty", "empty_limit_64"):
        assert recs[name]["rc"] == 0 and recs[name]["nout"] == 0 and recs[name]["launches"] == 0, recs[name]
