"""The host side of LEFT / SEMI / ANTI hash joins with a join filter, without a GPU (not gpu): libcbexec.so + the host code of
libcbgpu.so over the no-op runtime of tests/fake_runtime.py, a CUDA runtime that computes nothing (LD_PRELOADed into a
subprocess).  The filtered joins run to zero rows with launches, at 16 KB in batches; RIGHT,
FULL and NOT IN joins with a join filter are still refused; cbgpu_ht_probe_pairs refuses every malformed filter, a filter on
a join type that takes none and a SEMI join without one before any launch, stops between batches when interrupted, and
reports CBGPU_ERR_NOMEM for each of its device allocations failing in turn (filtered and unfiltered, one batch and 16), with
the next call clean.  Run as built and with libcbexec.so rebuilt under
AddressSanitizer + UBSan."""
from fake_runtime import run_worker

INVALID, UNSUPPORTED, NOMEM, INTERRUPTED = -2, -3, -5, -8


def _check(out):
    ran, refused = out["ran"], out["refused"]
    assert sorted(ran) == sorted("%s_dup%d_%dkb" % (j, d, m) for j in ("left", "semi", "anti") for d in (1, 3) for m in (0, 16))
    for name, r in ran.items():
        assert r["launches"] > 0, (name, r)
        if name.endswith("_16kb"):
            assert r["nbatch"] >= 4 and r["passes"] == r["nbatch"], (name, r)
        else:
            assert r["nbatch"] == 1 and r["passes"] == 0, (name, r)
        # a runtime that computes nothing: SEMI finds no partner, LEFT / ANTI rows are never counted either
        assert r["rows"] == 0, (name, r)
    assert sorted(refused) == sorted("%s_dup%d_%dkb" % (j, d, m) for j in ("right", "full", "notin") for d in (1, 3) for m in (0, 16))
    for name, r in refused.items():
        assert r["code"] == UNSUPPORTED and "extra join quals" in r["msg"], (name, r)
    for jt, r in out["abi_ok"].items():
        assert r["code"] == 0 and r["passes"] == 16 and r["launches"] > 16, (jt, r)
    for name, r in out["invalid"].items():
        assert r["code"] == INVALID and r["launches"] == 0 and r["npairs"] == 0 and r["passes"] == 0, (name, r)
    ai = out["abi_interrupt"]
    assert ai["code"] == INTERRUPTED and "canceling statement" in ai["msg"] and ai["polls"] == 3 and ai["passes"] == 2
    assert ai["npairs"] == 0 and ai["outer_idx"] is None
    oom = out["oom"]
    assert len(oom["codes"]) >= 8 and set(oom["codes"]) == {NOMEM}, oom
    assert set(oom["after"]) == {0}, oom


def test_pair_probe_with_and_without_filters_over_a_runtime_that_computes_nothing():
    _check(run_worker("host_join_filter_worker", "JOINFILTER")[0])


def test_pair_probe_with_and_without_filters_under_address_and_ub_sanitizers():
    _check(run_worker("host_join_filter_worker", "JOINFILTER", sanitized="exec")[0])
