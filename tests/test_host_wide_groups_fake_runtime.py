"""GROUP BY over up to eight columns without a GPU (not gpu): the host executor over the no-op runtime of tests/fake_runtime.py,
plain and with both libraries under AddressSanitizer + UBSan.  TPC-H Q10 (seven keys), Q18 (five keys, a HAVING aggregate under
a Hash), an 8-key plan and a numeric-key scan go through translation, kernel matching, launch and read-back on both kernel routes and under a 16 KB
budget; nine keys are refused with their code and message before any launch; every device allocation failing in turn is an
error that leaves nothing allocated."""
import pytest

from fake_runtime import run_worker

UNSUPPORTED, NOMEM = -3, -5


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_q10_q18_and_eight_keys_run_on_every_route(sanitized):
    recs = run_worker("host_wide_groups_worker", "WIDE", "runs", sanitized=sanitized, timeout=900)
    assert len(recs) == 16
    for r in recs:
        assert r["rc"] == 0 and r["launches"] > 0, r
        if r["name"] in ("q10", "q18") and not r["mem_kb"]:
            # the wide aggregate itself runs in the compiled probe chain unless the interpreter is forced; one table each
            # (the 8-key plan groups by nullable and float8 keys, which only the interpreter takes)
            assert r["agg_kernel"] == ("k_pipeline_generic" if r["generic"] else "k_probe_chain"), r
            assert r["agg_inits"] == (2 if r["name"] == "q18" else 1), r
        if r["name"] == "keys8":
            assert r["agg_kernel"] == "k_pipeline_generic", r


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_nine_keys_are_refused_before_any_launch(sanitized):
    (r,) = run_worker("host_wide_groups_worker", "WIDE", "refusal", sanitized=sanitized, timeout=600)
    assert r["rc"] == UNSUPPORTED and r["launches"] == 0, r
    assert "GROUP BY with 9 columns is beyond the GPU path's limit (8)" in r["msg"], r


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_failed_allocations_leave_nothing_allocated(sanitized):
    recs = {r["name"]: r for r in run_worker("host_wide_groups_worker", "WIDE", "frees", sanitized=sanitized, timeout=900)}
    assert set(recs) == {"q18", "keys8"}
    for r in recs.values():
        assert r["failed"] >= 3 and r["codes"] == [NOMEM] and r["leaks"] == [] and r["after"] == 0, r
