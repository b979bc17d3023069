"""HAVING without a GPU (not gpu): the host executor and cbgpu_having_select over the no-op runtime of tests/fake_runtime.py,
plain and with both libraries under AddressSanitizer + UBSan.  Q18 and the HAVING shapes of the capacity tests run on both
kernel routes and under a 16 KB budget (over the no-op runtime an aggregate has no groups, so HAVING keeps none and launches
nothing); the entry point's three kernels launch over a relation of 1000 groups; every shape the device path does not
evaluate is refused with its code and message before any launch; every device allocation of the entry point failing in turn
is an error that leaves nothing allocated."""
import pytest

from fake_runtime import run_worker

UNSUPPORTED, NOMEM = -3, -5


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_having_plans_run_on_every_route(sanitized):
    recs = run_worker("host_having_worker", "HAVING", "runs", sanitized=sanitized, timeout=900)
    assert len(recs) == 17
    for r in recs[:-1]:
        assert r["rc"] == 0 and r["rows"] == 0 and r["launches"] > 0, r
    (e,) = recs[-1:]
    assert e["rc"] == 0 and e["nsel"] == 0 and e["having"] == ["k_having_eval", "k_having_scan", "k_having_scatter"], e


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_unsupported_having_is_refused_before_any_launch(sanitized):
    recs = run_worker("host_having_worker", "HAVING", "refusals", sanitized=sanitized, timeout=600)
    assert [r["name"] for r in recs] == ["arithmetic", "mixed", "text", "dict_key", "in_list", "nine_aggs"]
    for r in recs:
        assert r["rc"] == UNSUPPORTED and r["launches"] == 0 and r["want"] in r["msg"], r


@pytest.mark.parametrize("sanitized", [None, "both"])
def test_failed_allocations_leave_nothing_allocated(sanitized):
    (r,) = run_worker("host_having_worker", "HAVING", "frees", sanitized=sanitized, timeout=600)
    assert r["failed"] >= 1 and r["codes"] == [NOMEM] and r["leaks"] == [] and r["after"] == 0, r
