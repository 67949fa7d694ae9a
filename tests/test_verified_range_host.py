"""dm_cache_open_verified_range on the CPU box: the engine compiled with g++ against the fake CUDA runtime
(tests/native/fake_cuda*: test infrastructure, its 'kernels' are the CPU oracle), soaked by tests/native/range_open_soak.cc
under ThreadSanitizer and ASan+UBSan, and the GPU module tests/test_gpu_verified_range.py run over the same build with a
small arena and small slabs."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS = os.path.join(ROOT, "demodel_b200", "csrc")
NATIVE = os.path.join(ROOT, "tests", "native")
ENGINE_SOURCES = [os.path.join(CS, f) for f in ("engine_core.cu", "engine_api.cu", "engine_cache.cu", "proxy_driver.cc",
                                                 "manifest.cc", "gunzip.cc")] + [os.path.join(NATIVE, "fake_cuda.cc")]


def _gxx(out, *flags, extra=(), shared=False):
    cmd = ["g++", "-std=c++17", "-O1", "-g", *flags, "-I", os.path.join(NATIVE, "fake_cuda"), "-pthread", "-o", str(out)]
    if shared:
        cmd += ["-shared", "-fPIC"]
    return subprocess.run(cmd + ["-x", "c++", *ENGINE_SOURCES, *extra], capture_output=True, text=True, timeout=600)


def test_range_open_soak_under_tsan_and_asan(tmp_path):
    """Reader threads open random ranges of blobs through shared ring loads, on an engine whose arena most blobs do not fit
    and on one without an HBM tier, and read them forward in random pieces, some stalling past the detach grace, some
    closing early, some trying a backward read or one outside their range, while other threads overwrite tier files in
    place, ingest, verify, remove, evict and set the disk limit.  Every byte a reader got is the one the load hashed, a
    last byte is only ever handed out after a verdict that matched, and at rest no slab, slot, HBM byte, descriptor or
    shared-load index entry is left over.  With no device jitter and with a random 0..300 us delay on every queued
    device operation."""
    ran = 0
    for name, flags in (("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])):
        exe = tmp_path / f"range_open_soak_{name}"
        build = _gxx(exe, *flags, extra=[os.path.join(NATIVE, "range_open_soak.cc")])
        if build.returncode != 0:
            if "sanitize" in build.stderr.lower() or "asan" in build.stderr.lower() or "tsan" in build.stderr.lower():
                continue                                          # this toolchain lacks that sanitizer runtime
            raise AssertionError(build.stderr[-3000:])
        env0 = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66", ASAN_OPTIONS="detect_leaks=0")
        runs = []
        for k, jitter in enumerate(("0", "300")):
            env = dict(env0, FAKE_CUDA_JITTER_US=jitter)
            args = [str(exe), "8", "6", str(tmp_path / f"cas_{name}_{k}")]
            runs.append((args, subprocess.Popen(args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)))
        for args, p in runs:
            text = p.communicate(timeout=900)[0]
            assert p.returncode == 0 and "RANGE OPEN SOAK OK" in text, " ".join(args) + "\n" + text[-4000:]
            assert "WARNING: ThreadSanitizer" not in text and "ERROR: AddressSanitizer" not in text and "runtime error" not in text, text[-4000:]
            ran += 1
    if ran == 0:
        pytest.skip("this g++ has no sanitizer runtime")


RUNNER = r"""
import os, sys, tempfile, pathlib, traceback
sys.path.insert(0, sys.argv[2])
import demodel_b200._lib as L
L.LIB_PATH = sys.argv[1]
import demodel_b200
import tests.test_gpu_verified_range as T
T.ARENA, T.RING, T.SLAB, T.BIG, T.SMALL_ARENA, T.IDLE = 16 << 20, 4 << 20, 64 << 10, 3 << 20, 1 << 20, 2 << 20
failed = ran = 0                                               # (the fake kernels are the scalar CPU oracle)
for name, fn in sorted(vars(T).items()):
    if not name.startswith("test_"):
        continue
    params = [{}]
    for m in getattr(fn, "pytestmark", []):
        if m.name == "parametrize":
            params = [{m.args[0]: v} for v in m.args[1]]
    for kw in params:
        try:
            fn(tmp_path=pathlib.Path(tempfile.mkdtemp(prefix="dm_range_")), **kw); print("ok   ", name, kw)
        except Exception:
            failed += 1; print("FAIL ", name, kw); traceback.print_exc()
        ran += 1
defined = sum(max([1] + [len(m.args[1]) for m in getattr(f, "pytestmark", []) if m.name == "parametrize"])
              for n, f in vars(T).items() if n.startswith("test_"))
print(f"VERIFIED RANGE MIRROR: {ran} ran, {failed} failed, {defined} defined")
sys.exit(1 if failed or ran < max(defined, 15) else 0)
"""


def test_gpu_verified_range_module_over_the_fake_runtime(tmp_path):
    """tests/test_gpu_verified_range.py against the engine built over the fake runtime, with a 1 MiB arena where the tests
    need a small one and 64 KiB slabs: the ctypes layer and the tests' own logic, every CPU run.  Not a parity claim."""
    lib = tmp_path / "libdemodel_b200_fake.so"
    build = _gxx(lib, shared=True)
    assert build.returncode == 0, build.stderr[-3000:]
    out = subprocess.run([sys.executable, "-c", RUNNER, str(lib), ROOT], capture_output=True, text=True, timeout=900,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and " 0 failed" in out.stdout, (out.stdout + out.stderr)[-4000:]
