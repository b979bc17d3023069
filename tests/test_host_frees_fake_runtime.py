"""A failing device-library call holds nothing it allocated (not gpu): libcbgpu.so and libcbexec.so over tests/native/fake_cudart.c,
a CUDA runtime that computes nothing and counts the device allocations still live (LD_PRELOADed into a subprocess, as
test_host_logic_fake_runtime.py does).  Every device allocation of each plan, and of each library call on its own, fails in turn:
the call reports CBGPU_ERR_NOMEM, a constructor leaves *out NULL, the live count is back where it was once the executor (or
the call's arguments) are freed, and the next run succeeds.  CBGPU_ERR_NOMEM is an answer a caller may act on (leave the work
to the CPU) and run the next query: memory a failed call kept would be missing from every query after it.  Run twice: as built,
and with both libraries rebuilt under AddressSanitizer + UBSan, where a double free on an error path shows."""
import json
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="needs the CUDA headers")

NOMEM = -5
CLUSTERS = ("q3_3seg", "q5_3seg", "q3_merge_gather_3seg")


@pytest.fixture(scope="module")
def fake(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakecuda")
    so = str(d / "libfakecudart.so")
    subprocess.check_call(["gcc", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
                           os.path.join(ROOT, "tests", "native", "fake_cudart.c")])
    return so


def _run(env):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "host_frees_worker.py")], capture_output=True, text=True,
                       timeout=1200, env=dict(os.environ, **env))
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("HOSTFREES ")]
    assert p.returncode == 0 and lines, (p.stdout[-2000:], p.stderr[-4000:])
    return json.loads(lines[0][len("HOSTFREES "):])


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


def test_failed_calls_leave_nothing_allocated(fake):
    _check(_run({"LD_PRELOAD": fake}))


def test_the_same_with_both_libraries_under_address_and_ub_sanitizers(fake, tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    if not (os.path.exists(nvcc) and os.path.exists(asan)):
        pytest.skip("needs nvcc and libasan")
    tree = tmp_path / "tree"
    shutil.copytree(os.path.join(ROOT, "cloudberry_b200", "csrc"), tree / "cloudberry_b200" / "csrc", ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(os.path.join(ROOT, "include"), tree / "include")
    san = "-Xcompiler -fsanitize=address -Xcompiler -fsanitize=undefined -Xcompiler -fno-omit-frame-pointer"
    subprocess.check_call(["make", "-s", "-j8", "-C", str(tree / "cloudberry_b200" / "csrc"), "../libcbgpu.so",
                           "ARCH=-gencode arch=compute_90a,code=sm_90a " + san])
    libdir = str(tree / "cloudberry_b200")
    src = os.path.join(ROOT, "cloudberry_b200", "csrc", "exec")
    subprocess.check_call(["gcc", "-O1", "-g", "-fPIC", "-shared", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                           "-o", os.path.join(libdir, "libcbexec.so")] +
                          [os.path.join(src, f) for f in ("cb_exec.c", "cb_numeric.c", "cb_aocs_load.c", "cb_tupser.c")] +
                          ["-L" + libdir, "-lcbgpu", "-Wl,-rpath," + libdir])
    _check(_run({"LD_PRELOAD": asan + ":" + fake, "ASAN_OPTIONS": "detect_leaks=0", "CB_TEST_LIBDIR": libdir}))
