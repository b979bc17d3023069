"""The host side of pair joins over a build side split into batches, without a GPU (not gpu): libcbexec.so + the host code of
libcbgpu.so over tests/native/fake_cudart.c, a CUDA runtime that computes nothing (LD_PRELOADed into a subprocess, as
test_host_logic_fake_runtime.py does).  RIGHT and FULL joins at a 16 KB operator memory return no rows (no kernel computes
anything) but walk every batch pass of the pair probe, the partition's read-back and the clean-up (INNER / LEFT ones run too,
through the N:1 passes: a runtime that computes nothing reports no duplicate build keys); the interrupt
callback stops the batch loop with CBGPU_ERR_INTERRUPTED; the single-pass pair probes refuse a multi-batch table.  Run as
built and with libcbexec.so rebuilt under AddressSanitizer + UBSan."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="needs the CUDA headers")

INVALID, INTERRUPTED = -2, -8


@pytest.fixture(scope="module")
def fake(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakecuda")
    so = str(d / "libfakecudart.so")
    subprocess.check_call(["gcc", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
                           os.path.join(ROOT, "tests", "native", "fake_cudart.c")])
    return d, so


def _run(env):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "host_batched_pairs_worker.py")], capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, **env))
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("BATCHEDPAIRS ")]
    assert p.returncode == 0 and lines, (p.stdout[-2000:], p.stderr[-4000:])
    assert "runtime error" not in p.stderr and "AddressSanitizer" not in p.stderr, p.stderr[-4000:]
    return json.loads(lines[0][len("BATCHEDPAIRS "):])


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
    sr = out["single_pass_refused"]
    assert sr["code"] == INVALID and "cbgpu_ht_probe_pairs_batched" in sr["msg"]
    ei = out["exec_interrupt"]
    assert ei["nbatch"] >= 4 and ei["polls_split"] - ei["polls_unsplit"] >= ei["nbatch"]
    assert set(ei["codes"]) == {INTERRUPTED} and len(ei["codes"]) == ei["polls_split"]
    assert ei["launches"] == sorted(ei["launches"]) and ei["launches"][-1] < ei["full_launches"]
    assert ei["rows_after"] == [0] * len(ei["codes"])


def test_batched_pair_joins_over_a_runtime_that_computes_nothing(fake):
    _, so = fake
    _check(_run({"LD_PRELOAD": so}))


def test_the_same_under_address_and_ub_sanitizers(fake):
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
