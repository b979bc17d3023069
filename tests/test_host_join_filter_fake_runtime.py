"""The host side of LEFT / SEMI / ANTI hash joins with a join filter, without a GPU (not gpu): libcbexec.so + the host code of
libcbgpu.so over tests/native/fake_cudart.c, a CUDA runtime that computes nothing (LD_PRELOADed into a subprocess, as
test_host_batched_pairs_fake_runtime.py does).  The filtered joins run to zero rows with launches, at 16 KB in batches; RIGHT,
FULL and NOT IN joins with a join filter are still refused; cbgpu_ht_probe_pairs refuses every malformed filter, a filter on
a join type that takes none and a SEMI join without one before any launch, stops between batches when interrupted, and
reports CBGPU_ERR_NOMEM for each of its device allocations failing in turn (filtered and unfiltered, one batch and 16), with
the next call clean.  Run as built and with libcbexec.so rebuilt under
AddressSanitizer + UBSan."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="needs the CUDA headers")

INVALID, UNSUPPORTED, NOMEM, INTERRUPTED = -2, -3, -5, -8


@pytest.fixture(scope="module")
def fake(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakecuda")
    so = str(d / "libfakecudart.so")
    subprocess.check_call(["gcc", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
                           os.path.join(ROOT, "tests", "native", "fake_cudart.c")])
    return d, so


def _run(env):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "host_join_filter_worker.py")], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, **env))
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("JOINFILTER ")]
    assert p.returncode == 0 and lines, (p.stdout[-2000:], p.stderr[-4000:])
    assert "runtime error" not in p.stderr and "AddressSanitizer" not in p.stderr, p.stderr[-4000:]
    return json.loads(lines[0][len("JOINFILTER "):])


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


def test_pair_probe_with_and_without_filters_over_a_runtime_that_computes_nothing(fake):
    _, so = fake
    _check(_run({"LD_PRELOAD": so}))


def test_pair_probe_with_and_without_filters_under_address_and_ub_sanitizers(fake):
    d, so = fake
    asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    if not os.path.exists(asan):
        pytest.skip("no libasan")
    libdir = str(d)
    src = os.path.join(ROOT, "cloudberry_b200", "csrc", "exec")
    os.symlink(os.path.join(ROOT, "cloudberry_b200", "libcbgpu.so"), os.path.join(libdir, "libcbgpu.so"))
    subprocess.check_call(["gcc", "-O1", "-g", "-fPIC", "-shared", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                           "-o", os.path.join(libdir, "libcbexec.so")] +
                          [os.path.join(src, f) for f in ("cb_exec.c", "cb_numeric.c", "cb_aocs_load.c", "cb_tupser.c")] +
                          ["-L" + libdir, "-lcbgpu", "-Wl,-rpath," + libdir])
    _check(_run({"LD_PRELOAD": asan + ":" + so, "ASAN_OPTIONS": "detect_leaks=0", "CB_TEST_LIBDIR": libdir}))
