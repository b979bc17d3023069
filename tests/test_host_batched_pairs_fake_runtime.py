"""The host side of pair joins over a build side split into batches, without a GPU (not gpu): libcbexec.so + the host code of
libcbgpu.so over the no-op runtime of tests/fake_runtime.py, a CUDA runtime that computes nothing (LD_PRELOADed into a
subprocess).  RIGHT and FULL joins at a 16 KB operator memory return no rows (no kernel computes
anything) but walk every batch pass of the pair probe, the partition's read-back and the clean-up (INNER / LEFT ones run too,
through the N:1 passes: a runtime that computes nothing reports no duplicate build keys); the interrupt
callback stops the batch loop with CBGPU_ERR_INTERRUPTED.  Run as built and with libcbexec.so rebuilt under AddressSanitizer +
UBSan."""
from fake_runtime import run_worker

INTERRUPTED = -8


def _check(out):
    for name, r in out["ran"].items():
        # nothing is computed: no rows; the build side was split and every batch got its pass
        assert r["rows"] == 0 and r["nbatch"] >= 4 and r["passes"] == r["nbatch"] and r["launches"] > r["passes"], (name, r)
    assert len(out["ran"]) == 16
    ai = out["abi_interrupt"]
    assert ai["code"] == INTERRUPTED and "canceling statement" in ai["msg"] and ai["polls"] == 3 and ai["passes"] == 2
    assert ai["launches"] < ai["full"]["launches"] and ai["full"]["passes"] == 16
    assert ai["npairs"] == 0 and ai["outer_idx"] is None         # a failed call leaves no pair list behind
    assert out["abi_after"]["passes"] == 16                       # and the table serves the next call
    ei = out["exec_interrupt"]
    assert ei["nbatch"] >= 4 and ei["polls_split"] - ei["polls_unsplit"] >= ei["nbatch"]
    assert set(ei["codes"]) == {INTERRUPTED} and len(ei["codes"]) == ei["polls_split"]
    assert ei["launches"] == sorted(ei["launches"]) and ei["launches"][-1] < ei["full_launches"]
    assert ei["rows_after"] == [0] * len(ei["codes"])


def test_pair_joins_in_batches_over_a_runtime_that_computes_nothing():
    _check(run_worker("host_batched_pairs_worker", "BATCHEDPAIRS")[0])


def test_pair_joins_in_batches_under_address_and_ub_sanitizers():
    _check(run_worker("host_batched_pairs_worker", "BATCHEDPAIRS", sanitized="exec")[0])
