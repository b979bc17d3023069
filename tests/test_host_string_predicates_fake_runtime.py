"""String predicates on the host side (not gpu): libcbgpu.so and libcbexec.so over tests/native/fake_cudart.c, a CUDA runtime
that computes nothing and counts the device allocations still live (LD_PRELOADed into subprocesses).

- tests/host_strings_worker.py: every refusal of LIKE / NOT LIKE / IN lists comes with its code and message before any kernel
  launch, also when a later predicate of the same scan is the one refused and when the predicate sits above a join; a
  character(n) column decoded from a file whose n was never declared refuses LIKE instead of matching it unpadded; accepted
  plans launch k_dict_like and run on k_pipeline_generic, on both routes, under a 16 KB budget and on a 3-segment cluster;
  every device allocation of the new library calls and plans failing in turn leaves nothing allocated.
- tests/native/inset_program.c: shapes the fused kernels take go to the generic kernel once they hold an INSET; INSET
  descriptors with a missing or malformed set, and join filters with an INSET, are refused before any launch."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="needs the CUDA headers")

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


@pytest.fixture(scope="module")
def fake(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakecuda")
    so = str(d / "libfakecudart.so")
    subprocess.check_call(["gcc", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
                           os.path.join(ROOT, "tests", "native", "fake_cudart.c")])
    return so


def test_executor_and_library_calls(fake):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "host_strings_worker.py")], capture_output=True, text=True,
                       timeout=1200, env=dict(os.environ, LD_PRELOAD=fake))
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("HOSTSTRINGS ")]
    assert p.returncode == 0 and lines, (p.stdout[-2000:], p.stderr[-4000:])
    out = json.loads(lines[0][len("HOSTSTRINGS "):])
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


def test_inset_descriptors(fake, tmp_path):
    exe = str(tmp_path / "inset_program")
    libdir = os.path.join(ROOT, "cloudberry_b200")
    subprocess.check_call(["gcc", "-O1", "-g", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "inset_program.c"), "-L" + libdir, "-lcbgpu", "-Wl,-rpath," + libdir])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, LD_PRELOAD=fake))
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    got = {}
    for ln in p.stdout.splitlines():
        name, code, launches, what = (ln.split(" ", 3) + [""])[:4]
        got[name] = (int(code), int(launches), what)
    assert set(got) == set(PROGRAMS)
    for name, (code, what) in PROGRAMS.items():
        c, n, w = got[name]
        assert c == code and (n > 0 if code == 0 else n == 0) and (w.startswith(what) if code == 0 else what in w), (name, got[name])
