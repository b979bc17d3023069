"""String predicates on the host side (not gpu): libcbgpu.so and libcbexec.so over the no-op runtime of tests/fake_runtime.py, a
CUDA runtime that computes nothing and counts the device allocations still live (LD_PRELOADed into subprocesses).

- tests/host_strings_worker.py: every refusal of LIKE / NOT LIKE / IN lists comes with its code and message before any kernel
  launch, also when a later predicate of the same scan is the one refused and when the predicate sits above a join; a
  character(n) column decoded from a file whose n was never declared refuses LIKE instead of matching it unpadded; accepted
  plans launch k_dict_like and run on k_pipeline_generic, on both routes, under a 16 KB budget and on a 3-segment cluster;
  every device allocation of the new library calls and plans failing in turn leaves nothing allocated.
- tests/native/inset_program.c: shapes the fused kernels take go to the generic kernel once they hold an INSET; INSET
  descriptors with a missing or malformed set, and join filters with an INSET, are refused before any launch."""
from fake_runtime import run_driver, run_worker

INVALID, UNSUPPORTED, NOMEM = -2, -3, -5
REFUSED = {"malformed_pattern": (INVALID, "must not end with escape character"),
           "no_dictionary": (UNSUPPORTED, "without a dictionary"),
           "not_a_string_column": (UNSUPPORTED, "without a dictionary"),
           "bpchar_n_not_declared": (UNSUPPORTED, "whose n was not declared"),
           "second_predicate_refused": (UNSUPPORTED, "without a dictionary"),
           "pattern_not_a_constant": (UNSUPPORTED, "other than a string constant"),
           "array_op_lt": (UNSUPPORTED, "array comparison with operator 12"),
           "array_eq_all": (UNSUPPORTED, "array comparison with operator 10 and useOr 0"),
           "array_ne_any": (UNSUPPORTED, "array comparison with operator 11 and useOr 1"),
           "null_element": (UNSUPPORTED, "NULL constants"),
           "null_string_element": (UNSUPPORTED, "NULL constants"),
           "mixed_elements": (UNSUPPORTED, "mixing string and other constants"),
           "five_string_predicates": (UNSUPPORTED, "more than 4 string predicates"),
           "text_constant_as_value": (UNSUPPORTED, "only taken as a LIKE pattern"),
           "above_a_join": (UNSUPPORTED, "only taken in the quals of a scan"),
           "texts_unsorted": (INVALID, "not above the one before it"),
           "texts_duplicate": (INVALID, "not above the one before it"),
           "texts_bpchar_trailing_blank": (INVALID, "trailing blanks"),
           "match_malformed_pattern": (INVALID, "must not end with escape character"),
           "match_bpchar_without_n": (INVALID, "does not fit the dictionary"),
           "match_varchar_with_n": (INVALID, "does not fit the dictionary"),
           "set_dict_bpchar_without_n": (INVALID, "does not fit the dictionary")}
ROUTES = ("scan_agg", "scan_agg_generic", "scan_agg_16kb", "build_side", "cluster_3seg")
PROGRAMS = {"q1": (0, "k_scan_agg_small<"), "q1_inset": (0, "k_pipeline_generic"), "q3": (0, "k_probe_chain"),
            "q3_inset": (0, "k_pipeline_generic"), "q3_inset_forced": (0, "k_pipeline_generic"),
            "inset_no_sets": (INVALID, "op 7: INSET of a code set the descriptor does not declare"),
            "inset_undeclared_set": (INVALID, "op 7: INSET of a code set the descriptor does not declare"),
            "inset_negative_set": (INVALID, "op 7: INSET of a code set the descriptor does not declare"),
            "too_many_sets": (INVALID, "declares 5 code sets"), "set_without_bits": (INVALID, "code set 0 malformed"),
            "set_negative_size": (INVALID, "code set 0 malformed"), "join_filter_inset": (INVALID, "join filter op 1")}


def test_executor_and_library_calls():
    out = run_worker("host_strings_worker", "HOSTSTRINGS", timeout=1200)[0]
    for name, (code, msg) in REFUSED.items():
        r = out["refused"][name]
        assert r["code"] == code and msg in r["msg"] and r["launches"] == 0, (name, r)
    assert out["refused"]["match_ok"] == {"code": 0, "msg": "", "launches": 1}
    for name in ROUTES:
        r = out["routes"][name]
        assert r["code"] == 0 and {"k_dict_like", "k_pipeline_generic"} <= set(r["kernels"]), (name, r)
    for name, r in list(out["calls"].items()) + list(out["plans"].items()):
        assert r["clean"]["code"] == 0 and r["clean"]["left"] == 0, (name, r["clean"])
        assert r["failed"] >= 1 and r["codes"] == [NOMEM], (name, r)
        assert r["leaks"] == [] and r["bad_out"] == [] and r["not_alloc"] == [], (name, r)
    assert out["calls"]["dict_from_texts"]["failed"] >= 4


def test_inset_descriptors():
    got = {name: (r["code"], r["launches"], r["what"]) for name, r in run_driver("inset_program").items()}
    assert set(got) == set(PROGRAMS)
    for name, (code, what) in PROGRAMS.items():
        c, n, w = got[name]
        assert c == code and (n > 0 if code == 0 else n == 0) and (w.startswith(what) if code == 0 else what in w), (name, got[name])
