"""Disk-backed streams (DM_F_DISK_DIRECT) on the CPU box: the engine compiled with g++ against the fake CUDA runtime
(tests/native/fake_cuda*: test infrastructure, its 'kernels' are the CPU oracle), soaked by tests/native/disk_direct_soak.cc
under ThreadSanitizer and ASan+UBSan, and the GPU module tests/test_gpu_disk_direct.py run over the same build."""
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


def test_disk_direct_soak_under_tsan_and_asan(tmp_path):
    """Several writer threads over a small arena (most bodies disk-backed): sequential and zero-copy writes, 2..16
    range parts in random order, aborts, wrong digests, flush + finish racing an abort, suspend -> destroy -> new
    engine -> resume, DM_F_NO_HBM_CAS | DM_F_DISK_DIRECT, and file writes failing under RLIMIT_FSIZE (DM_EIO, never
    a published file).  Then one disk-backed body at a time finishing while HBM writers keep an 8-slab ring busy, and
    16 disk-backed bodies at once over a 32-slab ring.  On a normal ring and a 4-slab one, with and without a random
    0..300 us delay on every queued device operation, and with 0..3 ms (the hash then trails the writers by far)."""
    ran = 0
    for name, flags in (("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])):
        exe = tmp_path / f"disk_soak_{name}"
        build = _gxx(exe, *flags, extra=[os.path.join(NATIVE, "disk_direct_soak.cc")])
        if build.returncode != 0:
            if "sanitize" in build.stderr.lower() or "asan" in build.stderr.lower() or "tsan" in build.stderr.lower():
                continue                                          # this toolchain lacks that sanitizer runtime
            raise AssertionError(build.stderr[-3000:])
        env0 = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66", ASAN_OPTIONS="detect_leaks=0")
        small = {"RIG_SLAB": "4096", "RIG_RING": "16384"}
        runs = []
        for k, (no_hbm, jitter, geo) in enumerate([(0, "0", {}), (1, "0", {}), (0, "300", {}), (1, "300", {}),
                                                   (0, "3000", {}), (0, "0", small), (1, "300", small)]):
            env = dict(env0, FAKE_CUDA_JITTER_US=jitter, **geo)
            args = [str(exe), "3", "8" if geo else "6", str(tmp_path / f"cas_{name}_{k}"), str(no_hbm)]
            runs.append((args, subprocess.Popen(args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)))
        for args, p in runs:
            text = p.communicate(timeout=600)[0]
            assert p.returncode == 0 and "DISK SOAK OK" in text, " ".join(args) + "\n" + text[-4000:]
            assert "WARNING: ThreadSanitizer" not in text and "ERROR: AddressSanitizer" not in text and "runtime error" not in text, text[-4000:]
            ran += 1
    if ran == 0:
        pytest.skip("this g++ has no sanitizer runtime")


RUNNER = r"""
import inspect, os, sys, tempfile, pathlib, traceback
sys.path.insert(0, sys.argv[2])
import demodel_b200._lib as L
L.LIB_PATH = sys.argv[1]
import demodel_b200
import tests.test_gpu_disk_direct as T
try:                                                  # DM_F_DISK_DIRECT without a disk tier
    demodel_b200.Engine(device=0, hbm_cas_bytes=1 << 20, flags=L.DM_F_DISK_DIRECT)
    sys.exit("DM_F_DISK_DIRECT without cas_dir was accepted")
except demodel_b200.DmError as ex:
    assert ex.code == L.DM_EINVAL, ex
T.ARENA, T.RING = 1 << 20, 4 << 20                    # bodies of a few MiB: the fake kernels are the scalar CPU oracle
failed = ran = 0
for name, fn in sorted(vars(T).items()):
    if not name.startswith("test_") or name == "test_four_gib_body":
        continue
    params = [{}]
    for m in getattr(fn, "pytestmark", []):
        if m.name == "parametrize":
            params = [{m.args[0]: v} for v in m.args[1]]
    for kw in params:
        kw = dict(kw, tmp_path=pathlib.Path(tempfile.mkdtemp(prefix="dm_disk_")))
        try:
            fn(**kw); print("ok   ", name, kw)
        except Exception:
            failed += 1; print("FAIL ", name, kw); traceback.print_exc()
        ran += 1
print(f"DISK MIRROR: {ran} ran, {failed} failed")
sys.exit(1 if failed or ran < 8 else 0)
"""


def test_gpu_disk_direct_module_over_the_fake_runtime(tmp_path):
    """tests/test_gpu_disk_direct.py (all but the 4 GiB body) against the engine built over the fake runtime, with a
    1 MiB arena: the ctypes layer and the tests' own logic, every CPU run.  Not a parity claim.  Also: the flag
    without cas_dir is DM_EINVAL."""
    lib = tmp_path / "libdemodel_b200_fake.so"
    build = _gxx(lib, shared=True)
    assert build.returncode == 0, build.stderr[-3000:]
    out = subprocess.run([sys.executable, "-c", RUNNER, str(lib), ROOT], capture_output=True, text=True, timeout=900,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and " 0 failed" in out.stdout, (out.stdout + out.stderr)[-4000:]
