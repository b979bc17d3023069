"""A failing device-library call holds nothing it allocated (not gpu): libcbgpu.so and libcbexec.so over the no-op
runtime of tests/fake_runtime.py, a CUDA runtime that computes nothing and counts the device allocations still live
(LD_PRELOADed into a subprocess).  Every device allocation of each plan, and of each library call on its own, fails in turn:
the call reports CBGPU_ERR_NOMEM, a constructor leaves *out NULL, the live count is back where it was once the executor (or
the call's arguments) are freed, and the next run succeeds.  CBGPU_ERR_NOMEM is an answer a caller may act on (leave the work
to the CPU) and run the next query: memory a failed call kept would be missing from every query after it.  Run twice: as built,
and with both libraries rebuilt under AddressSanitizer + UBSan, where a double free on an error path shows."""
from fake_runtime import run_worker

NOMEM = -5
CLUSTERS = ("q3_3seg", "q5_3seg", "q3_merge_gather_3seg")


def _check(out):
    plans, calls = out["plans"], out["calls"]
    assert set(plans) >= {"q1", "q3", "q5", "q1_generic", "q3_generic", "q5_generic", "q5_16kb", "orders_lineitem_16kb",
                          "right_join", "full_join", "join_filter_left", "join_filter_semi", "join_filter_anti", "having",
                          "limit_sort_agg", "ssb_q4_1"} | set(CLUSTERS)
    for name, r in list(plans.items()) + list(calls.items()):
        assert r["clean"]["code"] == 0 and r["clean"]["left"] == 0, (name, r["clean"])
        assert r["failed"] >= 1, name                                   # every sweep made something fail
        assert r["leaks"] == [], (name, r["leaks"])                     # [allocation that failed, allocations left behind]
        assert r["bad_out"] == [], (name, r["bad_out"])                 # *out set on failure, or the next run did not succeed
        # a cluster reports a segment's error with code -1 and that segment's message; each one names the failed allocation
        assert r["codes"] == ([-1] if name in CLUSTERS else [NOMEM]), (name, r["codes"])
        assert r["not_alloc"] == [], (name, r["not_alloc"][:3])
    for name in ("q3", "q5", "q5_16kb", "q3_3seg", "q5_3seg", "q3_merge_gather_3seg", "ssb_q4_1"):
        assert plans[name]["failed"] > 10, name
    for name in ("ht_build_16", "topn_10000", "rel_create_per_column", "aocs_apply_visimap", "aocs_decode_zstd1_int4_sorted"):
        assert calls[name]["failed"] >= 3, name
    assert calls["merge_sorted_runs"]["failed"] == 2                  # the run boundaries, then the order handed out
    assert len([k for k in calls if k.startswith("aocs_decode_")]) > 30
    # a status word reporting a device error at each 4-byte read-back of Q3 in turn: nothing left behind either
    assert out["status_word"]["raised"] >= 3 and out["status_word"]["leaks"] == []


def test_failed_calls_leave_nothing_allocated():
    _check(run_worker("host_frees_worker", "HOSTFREES", timeout=1200)[0])


def test_the_same_with_both_libraries_under_address_and_ub_sanitizers():
    _check(run_worker("host_frees_worker", "HOSTFREES", sanitized="both", timeout=1200)[0])
