"""Native (g++, no CUDA) randomized tests of the engine's host-only data structures: the HBM arena
allocator and the interval set behind range parts.  Runs on the CPU-only box."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_arena_and_interval_set_against_brute_force_models(tmp_path):
    exe = tmp_path / "test_host_util"
    src = os.path.join(ROOT, "tests", "native", "test_host_util.cc")
    flags = ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"]
    if subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", *flags, "-o", str(exe), src],
                      capture_output=True).returncode != 0:          # no sanitizer runtime: plain build
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-o", str(exe), src], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "host_util ok" in out.stdout


def test_manifest_parser_under_asan_ubsan(tmp_path):
    """200 000 mutated / random / truncated inputs through dm_manifest_parse built with
    -fsanitize=address,undefined: no over-read, no UB, only DM_OK or DM_EINVAL."""
    import pytest
    exe = tmp_path / "fuzz_manifest"
    src = os.path.join(ROOT, "tests", "native", "fuzz_manifest.cc")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                            "-o", str(exe), src], capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr.lower() or "sanitize" in build.stderr.lower()):
        pytest.skip("this g++ has no sanitizer runtime")
    assert build.returncode == 0, build.stderr[-2000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert "manifest fuzz ok" in out.stdout


def test_gunzip_under_asan_ubsan(tmp_path):
    """dm_gunzip (the manifest hook inflates `Content-Encoding: gzip` bodies with it) over real gzip / zlib streams
    with stored, fixed- and dynamic-Huffman blocks - and ~280 000 mutations of them - built with
    -fsanitize=address,undefined: only DM_OK / DM_EINVAL / DM_ENOMEM, no over-read, no over-write.  The
    reference's own cached gzip body (CONTRIBUTING.md:76-99) is one of the seeds."""
    import gzip
    import json
    import zlib
    import pytest
    exe = tmp_path / "fuzz_gunzip"
    src = os.path.join(ROOT, "tests", "native", "fuzz_gunzip.cc")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                            "-o", str(exe), src], capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr.lower() or "sanitize" in build.stderr.lower()):
        pytest.skip("this g++ has no sanitizer runtime")
    assert build.returncode == 0, build.stderr[-2000:]
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_fixture.json")))
    text = (b"{\"layers\":[" + b",".join(b"{\"digest\":\"sha256:%064x\",\"size\":%d}" % (i * 7919, i) for i in range(120)) + b"]}")
    fixed = zlib.compressobj(6, zlib.DEFLATED, 31, 8, zlib.Z_FIXED)
    seeds = [bytes.fromhex(fx["gzip_body_hex"]), gzip.compress(text, 9), gzip.compress(os.urandom(3000), 0), zlib.compress(text, 6),
             fixed.compress(text) + fixed.flush(), gzip.compress(b"", 6), gzip.compress(bytes(70000), 6)]
    paths = []
    for i, b in enumerate(seeds):
        paths.append(str(tmp_path / f"seed{i}.bin"))
        open(paths[-1], "wb").write(b)
    out = subprocess.run([str(exe), *paths], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert "gunzip fuzz ok" in out.stdout


def _build_rig(exe, *flags):
    build = subprocess.run([os.path.join(ROOT, "tests", "native", "build_rig.sh"), str(exe), *flags],
                           capture_output=True, text=True, timeout=600)
    return build


def test_engine_host_logic_soak_under_tsan_and_asan(tmp_path):
    """The whole engine (engine_*.cu + proxy driver + manifest) compiled with plain g++ against a fake CUDA
    runtime that is asynchronous like the real one (a worker thread per stream; copies and 'kernels' - the
    CPU oracle - run there; tests/native/fake_cuda*: test infrastructure, never part of the product), so
    that touching a slab, extent or job table before the event guarding it is a data race TSan reports;
    then soaked through the C-ABI by 6 threads mixing every
    ingest form, aborts, mismatches, cache reads, followers, evictions, checkpoint/resume — under
    ThreadSanitizer and under ASan+UBSan, with a tiny arena and ring so eviction and back-pressure are
    constantly exercised, in HBM-tier, disk-tier and verify-only modes.  No GPU involved: this is the
    regression net for the engine's locking and lifetime rules."""
    import pytest
    ran = 0
    for name, flags in (("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])):
        exe = tmp_path / f"rig_{name}"
        build = _build_rig(exe, *flags)
        if build.returncode != 0:
            if "sanitize" in build.stderr.lower() or "asan" in build.stderr.lower() or "tsan" in build.stderr.lower():
                continue                                          # this toolchain lacks that sanitizer runtime
            raise AssertionError(build.stderr[-3000:])
        base_env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66", ASAN_OPTIONS="detect_leaks=0")
        # the fourth run delays every queued operation by a random 0..300 us: real hardware's enqueue-to-execute gap
        # then: a 4-slab ring under 8 writers (parallel range parts and idle bodies pin partly filled slabs: the pump
        # must recall them, verify-only streams keeping their sub-block tail) - a stuck engine fails via the watchdog
        starved = {"RIG_SLAB": "4096", "RIG_RING": "16384", "RIG_DRV_RING": "262144"}
        for mode, jitter, geo in ((["3", "6"], "0", {}), (["3", "6", str(tmp_path / f"cas_{name}")], "0", {}),
                                  (["3", "6", "", "1"], "0", {}), (["3", "6"], "300", {}),
                                  (["3", "8"], "0", starved), (["3", "8", "", "1"], "0", starved),
                                  # 2 % of all host-to-device copies and launches fail: every fault must surface as
                                  # DM_ECUDA - never a wrong verdict, wrong bytes, a leak or a hang
                                  (["3", "6"], "0", {"FAKE_CUDA_FAIL_PPM": "20000"})):
            env = dict(base_env, FAKE_CUDA_JITTER_US=jitter, **geo)
            out = subprocess.run([str(exe), *mode], capture_output=True, text=True, timeout=300, env=env)
            text = out.stdout + out.stderr
            assert out.returncode == 0 and "ENGINE SOAK OK" in out.stdout, text[-4000:]
            assert "WARNING: ThreadSanitizer" not in text and "ERROR: AddressSanitizer" not in text and "runtime error" not in text, text[-4000:]
            ran += 1
        if name == "asan":
            # dm_engine_create's unwinding: fail the k-th device / pinned allocation, stream or event creation for a
            # spread of k (there are ~290 of them) - create must fail cleanly: no leak (LSan), no touch of freed memory
            ks = list(range(1, 13)) + list(range(13, 330, 11))
            seen_success = False
            for k in ks:
                env = dict(base_env, ASAN_OPTIONS="detect_leaks=1", FAKE_CUDA_FAIL_ALLOC_NTH=str(k))
                out = subprocess.run([str(exe), "create"], capture_output=True, text=True, timeout=120, env=env)
                text = out.stdout + out.stderr
                assert "Sanitizer" not in text and "runtime error" not in text, f"k={k}\n" + text[-3000:]
                assert out.returncode in (0, 2), f"k={k} rc={out.returncode}\n" + text[-2000:]
                seen_success = seen_success or out.returncode == 0
            assert seen_success, "the walk never got past the last allocation: extend ks"
    if ran == 0:
        exe = tmp_path / "rig_plain"                              # no sanitizer runtime at all: still run the soak
        build = _build_rig(exe)
        assert build.returncode == 0, build.stderr[-3000:]
        out = subprocess.run([str(exe), "3", "6"], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and "ENGINE SOAK OK" in out.stdout, (out.stdout + out.stderr)[-4000:]


def test_every_round_form_is_sha256_on_the_host(tmp_path):
    """sha256_round.cuh compiled as plain C++: each kernel round form (incl. the not-yet-default short chain)
    must reproduce the oracle's digests - the operation ORDER is what the forms differ in."""
    obj, exe = tmp_path / "oracle.o", tmp_path / "round_forms"
    subprocess.run(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "sha256_oracle.c"), "-o", str(obj)], check=True)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-fsanitize=undefined", "-fno-sanitize-recover=undefined",
                    os.path.join(ROOT, "tests", "native", "test_round_forms.cc"), str(obj), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ROUND FORMS OK" in out.stdout, out.stdout + out.stderr


def test_python_mirror_gpu_test_logic_and_bench_flow_over_the_fake_runtime(tmp_path):
    """The host-buffer tests of test_gpu_parity.py / test_manifest.py, run here against the engine built over the
    fake CUDA runtime (its 'kernels' are the CPU oracle): exercises the ctypes mirror and the tests' own logic on
    the CPU box, in a subprocess that patches the loader path for itself only.  Not a parity claim."""
    lib = tmp_path / "libdemodel_b200_fake.so"
    cs = os.path.join(ROOT, "demodel_b200", "csrc")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-pthread",
                            "-I", os.path.join(ROOT, "tests", "native", "fake_cuda"), "-o", str(lib), "-x", "c++",
                            os.path.join(cs, "engine_core.cu"), os.path.join(cs, "engine_api.cu"), os.path.join(cs, "engine_cache.cu"),
                            os.path.join(cs, "proxy_driver.cc"), os.path.join(cs, "manifest.cc"), os.path.join(cs, "gunzip.cc"),
                            os.path.join(ROOT, "tests", "native", "fake_cuda.cc")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stderr[-3000:]
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "native", "run_mirror_tests.py"), str(lib)],
                         capture_output=True, text=True, timeout=900)
    tail = (out.stdout + out.stderr)[-4000:]
    assert out.returncode == 0 and " 0 failed, leak=0" in out.stdout, tail
    # bench.py's whole control flow over the same build (numbers meaningless): it must reach its JSON line with
    # every key of the contract, in both arms
    import json
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "native", "run_bench_over_fake.py"), str(lib),
                          "--workload", "tiny", "--steps", "2", "--warmup", "1", "--no-probes"],
                         capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert out.returncode == 0, (out.stdout + out.stderr)[-4000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks"):
        assert key in line, key
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic", "int_issue"} <= set(line["roofline"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(line["cpu_baseline"])
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(line["e2e"])
    assert line["warmup"] >= 3 and line["gpu_launches"] > 0 and line["config"]["workload"] == "tiny"
    assert line["e2e"]["h2d_bytes_per_step"] == line["config"]["bytes_per_gpu_per_step"]
    # the host-cost probes (engine over null kernels) must keep working: they are how host-side work on the bulk and
    # tiny-body paths is measured without a GPU.  40 000 blobs: enough for the chunked-launch rule to apply.
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "native", "bulk_cost_probe.py"), str(lib), "40000", "1"],
                         capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.count("ns per blob") == 2, (out.stdout + out.stderr)[-2000:]


def test_sass_timing_model_ranks_the_short_chain_round_ahead(tmp_path):
    """tools/sass_sched.py on the built sm_90a kernels: ptxas' own ordering of the deep kernel's serial phase must come
    out at the model's 35 cycles per round, and the short-chain candidate must be predicted faster.  On an H100 SXM
    (1.98 GHz) the two measure 37.8 and 26.5 cycles per round (deep variants 0 and 7, 256 x 1 MiB): the model leaves
    out what the hardware adds (dispatch, LDS arrival), so it ranks round forms rather than predicting their time."""
    import re
    import shutil
    import pytest
    obj = os.path.join(ROOT, "demodel_b200", "csrc", "build", "sha256_kernels.o")
    if not (shutil.which("cuobjdump") and os.path.exists(obj)):
        pytest.skip("needs cuobjdump and the built kernel object")
    sass = tmp_path / "all.sass"
    with open(sass, "w") as f:
        subprocess.run(["cuobjdump", "-sass", obj], stdout=f, check=True, timeout=300)
    cyc = {}
    for v in (0, 4):
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_sched.py"), str(sass), f"deep_kernelILi{v}E"],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        cyc[v] = float(re.search(r"= ([0-9.]+) cycles per round", out.stdout).group(1))
    assert 33.5 <= cyc[0] <= 36.5, cyc           # model on sm_90a SASS: 35.0
    assert cyc[4] < cyc[0] - 2.0, cyc
