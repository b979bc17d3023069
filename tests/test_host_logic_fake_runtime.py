"""The host side of the product without a GPU (not gpu): libcbexec.so + the host code of libcbgpu.so run over a CUDA runtime
that computes nothing (the no-op runtime of tests/fake_runtime.py, LD_PRELOADed into a subprocess: zeroed host memory as
"device" memory, kernel launches are no-ops).  No result can come out of that - every query returns zero rows, which the test
asserts - but everything the host does around the kernels is exercised: Plan -> stream translation, pipeline program emission, the
specialised-kernel matcher, Motions inside a 3-segment cluster, launch bookkeeping, read-back, clean-up, the segment file loader's file handling (naming, EOFs, missing files), and the refusals
(HAVING, sorted aggregation, Sort without LIMIT, RIGHT join, numeric join keys, a scanrelid outside the range table) with the
error code and message a caller sees.  Run twice: as built, and with libcbexec.so rebuilt under AddressSanitizer + UBSan."""
import json
import os
import subprocess
import sys

from fake_runtime import ROOT, fake_cudart, run_worker

UNSUPPORTED, INVALID, NOMEM = -3, -2, -5


def _check(out):
    ran, refused = out["ran"], out["refused"]
    # partial-state (de)serialisation: every round trip exact, every truncation refused, random bytes (almost) never a state
    assert out["serialize"]["roundtrips"] == 300 and out["serialize"]["refused"] >= 300 * 5
    assert out["serialize"]["accepted_garbage"] < 30
    for name in ("q1", "q3", "q5", "q1_generic", "q3_generic", "q5_generic", "q1_3seg", "q3_3seg", "q5_3seg",
                 "ssb_q4_1", "ssb_q4_2", "ssb_q4_3", "q1_after_refusals", "having", "q3_tiny_memory",
                 "q3_merge_gather_3seg"):
        assert ran[name]["rows"] == 0, name            # nothing is computed on the host: no kernel, no rows
    for name in ("q1", "q3", "q5", "q1_3seg", "q3_3seg", "q5_3seg"):
        assert ran[name]["launches"] > 0
    assert ran["q3_3seg"]["launches"] > ran["q3"]["launches"]      # three segment executors and their Motions
    # outer joins go through the pair probe (count, scan, write, unmatched build rows); a PLAIN count over nothing is one row
    assert ran["right_join_runs"]["rows"] <= 1 and ran["right_join_runs"]["launches"] > 0 and ran["full_join_runs"]["launches"] > 0
    # a 16 KB operator memory: the build sides are split, every pass is a host loop iteration that launches (no-op) kernels
    assert ran["q3_tiny_memory"]["batches"] > 1 and ran["q3_tiny_memory"]["launches"] > ran["q3"]["launches"]
    assert ran["q3_merge_gather_3seg"]["launches"] > 0
    want = {"sorted_agg": (UNSUPPORTED, "hashed / plain"),
            "sort_without_limit": (UNSUPPORTED, "Sort without LIMIT"), "right_join": (UNSUPPORTED, "extra join quals"),
            "numeric_join_key": (UNSUPPORTED, "hash_numeric"), "bad_scanrelid": (INVALID, "scanrelid 9")}
    for name, (code, frag) in want.items():
        assert refused[name]["error"] is not None, name
        assert refused[name]["code"] == code and frag in refused[name]["error"], refused[name]
    for name in ("sorted_agg", "numeric_join_key", "bad_scanrelid"):
        assert refused[name]["launches"] == 0          # refused before anything reached the device
    # CHECK_FOR_INTERRUPTS between pipelines: the query stops early with its own code, the next one runs
    it = out["interrupt"]
    assert it["code"] == -8 and "canceling statement" in it["msg"] and it["launches"] < it["full"] and it["polls"] == 3 and it["rows_after"] == 0
    # the segment file loader: reference file naming, bytes past the recorded EOF ignored, and what cannot be read says why
    seg = out["segfile"]
    rows = seg["rows"]["int4_plain"]
    assert seg["loads"]["one_column"] == [rows, 0] and seg["loads"]["eof_zero"] == [0, 0]
    if "as_recorded" in seg["loads"]:
        assert seg["loads"]["as_recorded"] == [rows, 0]
    for name, frag in (("eof_beyond_file", "shorter than its recorded EOF"), ("eof_inside_a_block", "runs past the end of the file"),
                       ("missing_column_file", "16384.514"), ("missing_segno", "16384.9"), ("segno_out_of_range", "bad segment file name"),
                       ("visimap_same_range_twice", "two visimap entries"), ("visimap_misaligned_first_row", "multiple of 32768")):
        assert seg["errors"][name]["code"] == INVALID and frag in seg["errors"][name]["msg"], seg["errors"][name]
    assert "visimap_ok" in seg["loads"]
    # a full device: every allocation of Q5 failing in turn is CBGPU_ERR_NOMEM (the limit "inputs must fit HBM", which a caller may
    # answer by leaving the sub-tree to the CPU executor), never a crash, and the executor runs the query again afterwards
    assert out["oom"]["failed"] > 10 and out["oom"]["codes"] == [NOMEM] and out["oom"]["passed"] >= 3
    # an error the device reports in its status word (overflow, corrupt block, table full) reaches the caller with its code; a
    # word that makes no sense is an error too; the executor runs the query again afterwards
    de = out["device_errors"]
    assert de["raised"] >= 4 and {-4, -6, -5} <= set(de["codes"]) and all(-6 <= c < 0 for c in de["codes"])


def test_host_executor_over_a_runtime_that_computes_nothing():
    _check(run_worker("host_logic_worker", "HOSTLOGIC")[0])


def test_the_same_under_address_and_ub_sanitizers():
    _check(run_worker("host_logic_worker", "HOSTLOGIC", sanitized="exec")[0])


def test_storage_side_host_walk_under_sanitizers():
    """BOTH libraries rebuilt with AddressSanitizer + UBSan on their host code (the .cu files' host half through nvcc
    -Xcompiler): the plan shapes again, then cbgpu_aocs_decode_column's block header walk over every reference-written golden
    column file (plain, RLE / delta, zlib, zstd) and 40 damaged copies of each from exact-size buffers"""
    out = run_worker("host_logic_worker", "HOSTLOGIC", sanitized="both", env={"CB_TEST_AOCS_FUZZ": "40"})[0]
    _check(out)
    assert out["aocs_fuzz"]["calls"] > 1000 and out["aocs_fuzz"]["errors"] > 100


def test_bench_main_arm_control_flow(tmp_path):
    """bench.py's GPU arm from argument parsing to the JSON line, over the no-op runtime at a small scale factor: the numbers
    mean nothing (no kernel runs), the contract's keys and their bookkeeping do - steps, warm-up, launches counted, the e2e
    leg's byte counts, the q3 / q5 lines, one --dump-outputs file per timed query.  (The CPU legs have their own test,
    tests/test_bench_cpu.py.)"""
    dump = tmp_path / "out"
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--sf", "0.05", "--steps", "2", "--warmup", "3", "--no-cpu",
                        "--dump-outputs", str(dump)],
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, LD_PRELOAD=fake_cudart()), cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert p.returncode == 0 and len(lines) == 1, (p.stdout[-2000:], p.stderr[-3000:])
    line = json.loads(lines[0])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "roofline", "clocks", "gpu_launches", "e2e", "q3", "q5", "ssb", "result_check"):
        assert key in line, key
    # no golden rows exist for SF0.05: the line says so instead of claiming a check
    assert line["result_check"].startswith("unchecked") and line["q3"]["result_check"].startswith("unchecked")
    assert set(line["ssb"]["queries"]) == {"q4.1", "q4.2", "q4.3"}
    assert line["n_gpus"] == 1 and line["steps"] == 2 and line["warmup"] == 3 and line["unit"] == "rows/s"
    assert line["gpu_launches"] > 0 and "impl" not in line and "cpu_baseline" not in line
    rows = line["config"]["rows_per_gpu"]
    assert line["roofline"]["algorithmic_bytes_per_launch"] == 38 * rows and line["roofline"]["bound"] == "hbm"
    # host columns travel in the narrowest width holding their values (all zero over the no-op runtime: one byte each); the
    # decoded-width variant is measured beside it
    assert line["e2e"]["decoded_int64"]["h2d_bytes_per_step"] == 38 * rows and line["e2e"]["unit"] == "rows/s"
    assert line["e2e"]["h2d_bytes_per_step"] == 7 * rows and line["e2e"]["bytes_per_row_shipped"] == 7
    for q in ("q3", "q5"):
        assert line[q]["gpu_launches_per_step"] > 0 and line[q]["roofline"]["algorithmic_bytes"] > 0 and line[q]["steps"] == 2
    assert line["ssb"]["steps"] == 2
    assert sorted(os.listdir(dump)) == ["q1.npy", "q3.npy", "q5.npy", "ssb_q4_1.npy", "ssb_q4_2.npy", "ssb_q4_3.npy"]


def test_bench_result_check_bites(tmp_path):
    """with golden rows for the configuration at hand, a run whose kernels compute nothing must FAIL: bench.py prints its line with
    result_check = MISMATCH and exits 1"""
    import multiprocessing as mp
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_bench_golden as G
    with mp.Pool(2) as pool:
        gold = {"q1_sf0.05": G.run_q1(pool, 0.05, 1), "q3_sf0.05": G.run_q3(pool, 0.05), "q5_sf0.05": G.run_q5(pool, 0.05)}
    path = tmp_path / "gold.json"
    path.write_text(json.dumps(gold))
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--sf", "0.05", "--steps", "2", "--warmup", "3", "--no-cpu", "--no-e2e", "--no-ssb"],
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, LD_PRELOAD=fake_cudart(), CBGPU_BENCH_GOLDEN=str(path)), cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert p.returncode == 1 and len(lines) == 1, (p.returncode, p.stdout[-2000:], p.stderr[-2000:])
    line = json.loads(lines[0])
    assert line["result_check"].startswith("MISMATCH") and line["q5"]["result_check"].startswith("MISMATCH")
    assert "result_check FAILED" in p.stderr


def test_smoke_cannot_pass_without_real_kernels():
    """__graft_entry__.smoke() compares the device's rows with the oracle's and the reference's expected rows: over a runtime
    whose kernels do nothing it must fail - it is a check of results, not of plumbing"""
    p = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, LD_PRELOAD=fake_cudart()), cwd=ROOT)
    assert p.returncode != 0 and "AssertionError" in p.stderr, (p.stdout[-500:], p.stderr[-1500:])
    assert "smoke ok" not in p.stdout
