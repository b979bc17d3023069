"""The postfix program of a pipeline descriptor, checked on the host (not gpu): tests/native/pipeline_program.c builds CbPipeline
descriptors in C and calls cbgpu_pipeline_run over the no-op runtime of tests/fake_runtime.py, a CUDA runtime that computes
nothing (LD_PRELOADed).  Every malformed program is refused with its code before anything is
launched; a program whose stack reaches exactly CBP_STACK values runs; each valid shape goes to the kernel that fuses it, or to
the generic kernel when a matcher must decline it (float8 order keys, a qual behind a probe, a NE qual, an empty qual range).
Run twice: as built, and with libcbgpu.so and the driver rebuilt under AddressSanitizer + UBSan."""
import re

from fake_runtime import run_driver

INVALID, UNSUPPORTED = -2, -3
SMALL_AGG, PROBE_CHAIN, GENERIC = "k_scan_agg_small<", "k_probe_chain", "k_pipeline_generic"

REFUSED = {"load_missing_column": INVALID, "load_negative_column": INVALID, "dup_out_of_range": INVALID, "dup_negative": INVALID,
           "underflow_binary": INVALID, "underflow_compare": INVALID, "underflow_unary": INVALID, "underflow_f8ord": INVALID,
           "underflow_filter": INVALID, "underflow_pop": INVALID, "probe_bad_index": INVALID, "probe_negative_index": INVALID,
           "probe_too_few_keys": INVALID, "end_before_last": INVALID, "unknown_opcode": INVALID, "internal_opcode": INVALID,
           "negative_opcode": INVALID, "no_end": INVALID, "depth_49": UNSUPPORTED}
# the op a refusal names: the first of a program that breaks at once, the second of one that breaks after one LOAD
AT_FIRST = {"underflow_unary", "underflow_f8ord", "underflow_filter", "underflow_pop", "probe_too_few_keys"}
AT_OP = {name: 0 if name in AT_FIRST else 1 for name in REFUSED if name not in ("no_end", "depth_49")}
ROUTES = {"q1": SMALL_AGG, "q1_f8ord": GENERIC, "q1_ne": GENERIC, "q1_empty": GENERIC, "q1_empty_top": GENERIC,
          "q1_wide_const": GENERIC, "q3": PROBE_CHAIN, "q3_f8ord": GENERIC, "q3_qual_behind_probe": GENERIC, "q3_ne": GENERIC,
          "q3_empty": GENERIC, "q3_between": PROBE_CHAIN, "q3_between_empty": GENERIC, "q3_byte_qual": PROBE_CHAIN,
          "q3_byte_empty": GENERIC}


def _check(out):
    assert set(out) == set(REFUSED) | set(ROUTES) | {"depth_48"}, sorted(out)
    for name, code in REFUSED.items():
        r = out[name]
        assert r["code"] == code and r["launches"] == 0, (name, r)
        if name in AT_OP:
            assert re.search(r"\bop %d\b" % AT_OP[name], r["what"]), (name, r)
    assert out["depth_48"]["code"] == 0 and out["depth_48"]["launches"] > 0, out["depth_48"]
    for name, kernel in ROUTES.items():
        r = out[name]
        assert r["code"] == 0 and r["launches"] > 0 and r["what"].startswith(kernel), (name, r)


def test_pipeline_programs_over_a_runtime_that_computes_nothing():
    _check(run_driver("pipeline_program"))


def test_the_same_under_address_and_ub_sanitizers():
    _check(run_driver("pipeline_program", sanitized=True))
