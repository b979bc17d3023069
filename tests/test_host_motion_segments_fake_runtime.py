"""How many segments a Motion of the in-process cluster takes, without a GPU (not gpu): libcbexec.so built under AddressSanitizer +
UBSan over the no-op runtime of tests/fake_runtime.py.  A hash Motion keeps its per-destination bases, capacities and counts in
64-entry arrays (the sink's and the staged pass's), so on 65 segments it must be refused with CBGPU_ERR_UNSUPPORTED before any of
them is written, on the cluster's path as on an interconnect's: no sanitizer report.  64 segments are accepted, and a Gather or
a Broadcast, which routes nothing, runs on 65."""
from fake_runtime import run_worker

UNSUPPORTED = -3


def test_hash_motion_over_65_segments_is_refused_and_64_run():
    recs = {(r["nsegs"], r["case"]): r for r in run_worker("host_motion_segments_worker", "MOTIONSEGS", sanitized="exec")}
    assert set(recs) == {(s, c) for s in (64, 65) for c in ("hash", "hash_two_keys", "gather", "broadcast")}
    for case in ("hash", "hash_two_keys"):
        r = recs[(65, case)]
        assert r["code"] == UNSUPPORTED and "more than 64 segments (65)" in r["msg"], r
    for key, r in recs.items():
        if key[0] == 64 or key[1] in ("gather", "broadcast"):
            # nothing is computed over the no-op runtime: no rows, but every sender slice launched its kernel
            assert r["code"] == 0 and r["rows"] == 0 and r["launches"] >= key[0], (key, r)
