"""The host loop of the device top-N (cbgpu_topn, ORDER BY ... LIMIT n with n <= 64) without a GPU (not gpu): libcbgpu.so over
the no-op runtime of tests/fake_runtime.py, a CUDA runtime that computes nothing (LD_PRELOADed into a subprocess).  Every key
reads back as constant there, so the threshold selection gives up on each key and every call goes to the tournament, the host
loop of k_topn passes.  Every LIMIT from 1 to 64 must return, over 4097, 10 000 and 10^6 rows, with a number of launches
logarithmic in the rows: a pass that does not shrink its input would loop forever.  The refusals (key count, LIMIT range, bad key
column, nullable and float8 keys) come with their code and message and before any launch; an empty relation gives no rows."""
import math

import pytest

from fake_runtime import run_worker

INVALID, UNSUPPORTED = -2, -3


@pytest.mark.parametrize("n", [4097, 10000, 10**6])
def test_every_limit_returns_in_logarithmic_launches(n):
    # a pass that does not shrink its input never returns: the timeout fails the test with the last call that returned
    recs = run_worker("host_topn_worker", "TOPN", "calls", n, timeout=60)
    assert [(r["nkeys"], r["limit"]) for r in recs] == [(k, lim) for k in (1, 4) for lim in range(1, 65)]
    for r in recs:
        assert r["rc"] == 0, r
        # the no-op runtime reads back zeroed indices: row 0, a row all the same, so every slot is filled
        assert r["nout"] == r["limit"], r
        # per key one k_topn_min + k_topn_kth (every key is constant here), then tournament passes that at least halve the input
        assert 0 < r["launches"] <= math.ceil(math.log2(n)) + 2 * r["nkeys"] + 2, r


def test_refusals_come_before_any_launch():
    recs = {r["name"]: r for r in run_worker("host_topn_worker", "TOPN", "refusals", timeout=60)}
    want = {"nkeys_0": (UNSUPPORTED, "1..4 sort keys and LIMIT <= 64"), "nkeys_5": (UNSUPPORTED, "1..4 sort keys and LIMIT <= 64"),
            "limit_0": (UNSUPPORTED, "got 0"), "limit_65": (UNSUPPORTED, "got 65"),
            "key_col_3": (INVALID, "bad key column 3"), "key_col_neg": (INVALID, "bad key column -1"),
            "float8_key": (UNSUPPORTED, "float8 key"), "nullable_key": (UNSUPPORTED, "nullable sort key")}
    for name, (code, frag) in want.items():
        r = recs[name]
        assert r["rc"] == code and frag in r["msg"] and r["launches"] == 0, r
    for name in ("empty", "empty_limit_64"):
        assert recs[name]["rc"] == 0 and recs[name]["nout"] == 0 and recs[name]["launches"] == 0, recs[name]
