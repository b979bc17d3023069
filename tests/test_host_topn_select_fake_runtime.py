"""The host side of the device top-N for any LIMIT (cbgpu_topn_select, csrc/agg.cu) without a GPU (not gpu): libcbgpu.so over
the no-op runtime of tests/fake_runtime.py (LD_PRELOADed into a subprocess), plain and with both libraries under AddressSanitizer
+ UBSan.  Every key reads back constant there, so no digit can vary and a call is the image pass and k_tsel_finish: every LIMIT
up to 10^6, over up to 10^6 rows, returns min(limit, rows) indices within the launch bound (two plus six per varying digit).  The
refusals (key count, LIMIT, bad key column, a float8 order over a narrower column, a NULL source that is not an int8 column) come
with their code and message and before any launch, and every device allocation failing in turn leaves nothing allocated."""
import pytest

from fake_runtime import run_worker

INVALID, UNSUPPORTED, NOMEM = -2, -3, -5
LIMITS = [1, 64, 65, 100, 4096, 10**6]
MAX_DIGITS = 4 * 9              # per key: a NULL digit and eight 8-bit digits


@pytest.mark.parametrize("sanitized", [None, "both"])
@pytest.mark.parametrize("n", [1, 65, 10**6])
def test_every_limit_returns_its_rows_within_the_launch_bound(n, sanitized):
    recs = run_worker("host_topn_select_worker", "TSEL", "calls", n, sanitized=sanitized, timeout=600)
    assert [(r["nkeys"], r["limit"]) for r in recs] == [(k, lim) for k in (1, 4) for lim in LIMITS]
    for r in recs:
        assert r["rc"] == 0, r
        assert r["nout"] == min(r["limit"], n), r
        assert r["launches"] <= 2 + 6 * MAX_DIGITS, r
        assert r["launches"] == 2, r        # k_tsel_image, k_tsel_finish: no digit varies here


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_refusals_come_before_any_launch(sanitized):
    recs = {r["name"]: r for r in run_worker("host_topn_select_worker", "TSEL", "refusals", sanitized=sanitized, timeout=600)}
    want = {"nkeys_0": (UNSUPPORTED, "1..4 sort keys (0 keys)"), "nkeys_5": (UNSUPPORTED, "1..4 sort keys (5 keys)"),
            "limit_0": (UNSUPPORTED, "LIMIT >= 1 (got 0)"), "limit_neg": (UNSUPPORTED, "LIMIT >= 1 (got -1)"),
            "key_col_4": (INVALID, "bad key column 4"), "key_col_neg": (INVALID, "bad key column -1"),
            "key_128bit": (INVALID, "key column 3 is not 1, 4 or 8 bytes wide"),
            "float8_on_int4": (INVALID, "float8 order over a column narrower than 8 bytes (column 2)"),
            "null_col_float8": (INVALID, "NULL-source column 1 is not an int8 column"),
            "null_col_int4": (INVALID, "NULL-source column 2 is not an int8 column"),
            "null_col_out": (INVALID, "NULL-source column 7 is not an int8 column"),
            "null_source_bad": (INVALID, "unknown NULL source 9")}
    for name, (code, frag) in want.items():
        r = recs[name]
        assert r["rc"] == code and frag in r["msg"] and r["launches"] == 0, r
    for name in ("empty", "empty_limit_10e6"):
        assert recs[name]["rc"] == 0 and recs[name]["nout"] == 0 and recs[name]["launches"] == 0, recs[name]


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_failed_allocations_leave_nothing_allocated(sanitized):
    n = 100000
    recs = {r["name"]: r for r in run_worker("host_topn_select_worker", "TSEL", "frees", n, sanitized=sanitized, timeout=600)}
    for name, limit in (("frees_limit_100", 100), ("frees_limit_%d" % n, n)):
        r = recs[name]
        assert r["failed"] >= 3 and r["codes"] == [NOMEM] and r["leaks"] == [], r
        assert r["nout"] == limit, r
