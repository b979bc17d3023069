"""The no-op CUDA runtime the host tests run over (tests/native/fake_cudart.c), the libraries built under AddressSanitizer +
UBSan, and the two ways to run a program over them.  Not a test by itself.

Each artefact is built at most once per pytest process, under one temporary directory removed at exit.  The libraries are built
by the product's Makefile in a copy of the tree, so they are the libraries the product builds and the product's own are never
overwritten.  Every run must exit 0 and print its tag line, and its stderr must hold no sanitizer report: a report the sanitized
code did not abort on fails the run as well."""
import atexit
import functools
import json
import logging
import os
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT = os.path.join(ROOT, "cloudberry_b200")
CUDA_INC = "/usr/local/cuda/include"
CC = "gcc"          # handed to make as well: the environment's CC may name a compiler without the sanitizer runtimes
SANITIZE = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"]
REPORTS = ("runtime error", "Sanitizer")       # UBSan's "runtime error: ...", AddressSanitizer, LeakSanitizer, ...

log = logging.getLogger(__name__)


@functools.cache
def _tmp():
    d = tempfile.mkdtemp(prefix="cb_fake_runtime_")
    atexit.register(shutil.rmtree, d, True)
    return d


def _build(*cmd):
    log.info("build: %s", " ".join(cmd))
    subprocess.check_call(cmd)


@functools.cache
def _libasan():
    path = subprocess.check_output([CC, "-print-file-name=libasan.so"], text=True).strip()
    return path if os.path.exists(path) else None


@functools.cache
def fake_cudart():
    """the path of the no-op runtime, to LD_PRELOAD"""
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")):
        pytest.skip("needs the CUDA headers")
    so = os.path.join(_tmp(), "libfakecudart.so")
    _build(CC, "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-I" + CUDA_INC, "-o", so,
           os.path.join(ROOT, "tests", "native", "fake_cudart.c"))
    return so


@functools.cache
def sanitized_libdir(which):
    """a directory holding libcbexec.so built under ASan + UBSan and the libcbgpu.so it loads: for which="exec" a copy of the
    product's, for which="both" one whose host code is built under ASan + UBSan too (nvcc -Xcompiler)"""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not _libasan() or (which == "both" and not os.path.exists(nvcc)):
        pytest.skip("needs nvcc and libasan" if which == "both" else "no libasan")
    tree = os.path.join(_tmp(), which)
    shutil.copytree(os.path.join(PRODUCT, "csrc"), os.path.join(tree, "cloudberry_b200", "csrc"), ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tree, "include"))
    libdir = os.path.join(tree, "cloudberry_b200")
    make = ["make", "-s", "-j8", "-C", os.path.join(libdir, "csrc"), "CC=" + CC, "EXEC_CFLAGS=-O1 " + " ".join(SANITIZE)]
    if which == "both":
        san = ("-Xcompiler -fsanitize=address -Xcompiler -fsanitize=undefined -Xcompiler -fno-omit-frame-pointer"
               " -Xcompiler -fno-sanitize-recover=undefined")
        _build(*make, "ARCH=-gencode arch=compute_90a,code=sm_90a " + san, "../libcbgpu.so", "../libcbexec.so")
    else:
        # make must not rebuild the copied libcbgpu.so (-o); the executor's rpath $ORIGIN loads it
        shutil.copy(os.path.join(PRODUCT, "libcbgpu.so"), libdir)
        _build(*make, "-o", "../libcbgpu.so", "../libcbexec.so")
    return libdir


def _env(sanitized):
    if sanitized is None:
        return {"LD_PRELOAD": fake_cudart()}
    return {"LD_PRELOAD": _libasan() + ":" + fake_cudart(), "ASAN_OPTIONS": "detect_leaks=0",
            "CBGPU_LIBDIR": sanitized_libdir(sanitized)}


def _run(cmd, tag, env, timeout):
    """the stdout lines starting with tag, tag removed"""
    try:
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **env))
    except subprocess.TimeoutExpired as e:
        out = e.stdout.decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
        done = [ln for ln in out.splitlines() if ln.startswith(tag)]
        pytest.fail("%s did not finish within %ds; last line printed (the last call that returned): %s"
                    % (" ".join(cmd), timeout, done[-1] if done else "none"))
    lines = [ln[len(tag):] for ln in p.stdout.splitlines() if ln.startswith(tag)]
    assert p.returncode == 0 and lines, (p.returncode, p.stdout[-2000:], p.stderr[-4000:])
    assert not any(r in p.stderr for r in REPORTS), p.stderr[-4000:]
    return lines


def run_worker(worker, tag, *args, sanitized=None, env=None, timeout=600):
    """the JSON objects the Python worker tests/<worker>.py prints after `tag `, run with args over the no-op runtime and the
    product's libraries, or with sanitized="exec" / "both" over sanitized_libdir(sanitized); env: more environment"""
    cmd = [sys.executable, os.path.join(ROOT, "tests", worker + ".py")] + [str(a) for a in args]
    return [json.loads(ln) for ln in _run(cmd, tag + " ", dict(_env(sanitized), **(env or {})), timeout)]


@functools.cache
def _driver(name, sanitized):
    libdir = sanitized_libdir("both") if sanitized else PRODUCT
    exe = os.path.join(_tmp(), name + ("_sanitized" if sanitized else ""))
    _build(CC, "-O1", "-g", "-Wall", "-Werror", *(SANITIZE if sanitized else []), "-I" + os.path.join(ROOT, "include"), "-o", exe,
           os.path.join(ROOT, "tests", "native", name + ".c"), "-L" + libdir, "-lcbgpu", "-Wl,-rpath," + libdir)
    return exe


def run_driver(name, sanitized=False, timeout=600):
    """the table the C driver tests/native/<name>.c prints, one '<case> <code> <launches> <kernel or message>' line per case, as
    {case: {"code", "launches", "what"}}; run over the no-op runtime and the product's libcbgpu.so, or with sanitized=True built
    under ASan + UBSan and run over sanitized_libdir("both")"""
    env = _env("both" if sanitized else None)
    out = {}
    for ln in _run([_driver(name, sanitized)], "", env, timeout):
        case, code, launches, what = (ln.split(" ", 3) + [""])[:4]
        out[case] = {"code": int(code), "launches": int(launches), "what": what}
    return out
