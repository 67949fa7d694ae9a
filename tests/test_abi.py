"""C-ABI checks that need no GPU: the library loads, exports every symbol the
header declares, and refuses (loudly) to run the hash path without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import demodel_b200
from demodel_b200 import _lib
from demodel_b200.shard import owner_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "demodel_b200.h")


def _declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dm_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = demodel_b200.load()
    names = _declared_symbols()
    assert len(names) >= 25
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/demodel_b200.h but not exported"
    # and the ctypes table covers exactly the header
    assert sorted(_lib.SIGNATURES) == names


def test_abi_version_and_struct_layout():
    lib = demodel_b200.load()
    assert lib.dm_abi_version() == 2
    assert C.sizeof(_lib.DmConfig) == 48        # matches the C layout on LP64
    assert C.sizeof(_lib.DmStats) == 25 * 8


def test_strerror_covers_all_codes():
    lib = demodel_b200.load()
    seen = {lib.dm_strerror(c).decode() for c in range(0, -9, -1)}
    assert len(seen) == 9 and "unknown error" not in seen
    assert lib.dm_strerror(-99).decode() == "unknown error"


def test_shard_of_matches_python_router():
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 4, 8, 7):
        for _ in range(200):
            d = rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()
            assert demodel_b200.shard_of(d, n) == owner_of(d, n)
    # powers of two reduce to the leading bits of digest[0] (SURVEY.md §8e)
    for b in range(256):
        d = bytes([b]) + bytes(31)
        assert demodel_b200.shard_of(d, 4) == b >> 6
        assert demodel_b200.shard_of(d, 8) == b >> 5


def test_rejects_bad_config():
    lib = demodel_b200.load()
    cfg = _lib.DmConfig()
    cfg.struct_size = 4                           # wrong ABI guard
    h = C.c_void_p()
    assert lib.dm_engine_create(C.byref(cfg), C.byref(h)) == _lib.DM_EINVAL
    assert not h.value


def test_no_cpu_fallback_without_a_device():
    lib = demodel_b200.load()
    if lib.dm_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(demodel_b200.DmError) as ei:
        demodel_b200.Engine(device=0, hbm_cas_bytes=1 << 20)
    assert ei.value.code == demodel_b200.DM_ENODEV


def test_product_generator_matches_oracle_generator(oracle):
    # host half of the synthetic-bytes generator (pure CPU, no device needed)
    seed = 0xDE40DE1
    for blob, off, n in [(0, 0, 4096), (3, 5, 1000), (9, 8, 64), (2, 1 << 33, 777), (1, 123457, 33)]:
        assert np.array_equal(demodel_b200.synth_fill_host(seed, blob, off, n), oracle.blob(seed, blob, off, n))


def test_header_is_plain_c(tmp_path):
    """The boundary must be bindable from cgo: the header has to compile as C99, not only as C++."""
    import subprocess
    src = tmp_path / "use_header.c"
    src.write_text('#include "demodel_b200.h"\n'
                   'int main(void) { dm_config c; dm_stats s; dm_checkpoint k; dm_layer l;\n'
                   '  (void)c; (void)s; (void)k; (void)l; return (int)sizeof(dm_config) == 48 ? 0 : 1; }\n')
    exe = tmp_path / "use_header"
    subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    "-o", str(exe), str(src)], check=True)
    assert subprocess.run([str(exe)]).returncode == 0


def test_reference_arm_runs_without_a_gpu():
    """bench.py --impl reference is the CPU arm: it must run (and print the contract's keys) on a box
    with no GPU at all."""
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "tiny",
                          "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().split("\n")[-1])
    assert line["impl"] == "reference" and line["unit"] == "GB/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"] == {"value": line["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["higher_is_better"] is True and line["config"]["workload"] == "tiny"


def test_kernel_selection_rule_and_bench_mirror():
    """streams_per_warp_for(): monotone, powers of two; while there are sub-partitions to spare every group of S streams
    gets a warp PAIR (at most 264 groups, so up to 4224 streams), then one warp per sub-partition (528) at S = 16, then
    a lane per stream - deep (S = 1, paired) for the BASELINE 256-stream config; bench.py's report label mirrors it."""
    import importlib.util
    lib = demodel_b200.load()
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    prev = 0
    edges = [264, 265, 528, 529, 1056, 1057, 2112, 2113, 4224, 4225, 8448, 8449]
    for n in list(range(1, 20000, 37)) + [256, 135168, 1 << 31] + edges:
        spw = lib.dm_streams_per_warp(n)
        assert spw in (1, 2, 4, 8, 16, 32)
        groups = (n + spw - 1) // spw
        assert spw == 32 or groups <= 528
        assert spw in (16, 32) or groups <= 264                         # S < 16 is only ever chosen with room for pairs
        label = bench._kernel_for(n)
        assert (f"{spw} stream" in label) and (("pair" in label) == (spw < 32 and groups <= 264))
    for n in sorted(list(range(1, 20000, 37)) + edges):
        spw = lib.dm_streams_per_warp(n)
        assert spw >= prev
        prev = spw
    assert lib.dm_streams_per_warp(256) == 1 and lib.dm_streams_per_warp(8449) == 32 and lib.dm_streams_per_warp(4096) == 16
    assert lib.dm_streams_per_warp(264) == 1 and lib.dm_streams_per_warp(265) == 2 and lib.dm_streams_per_warp(528) == 2
    assert lib.dm_streams_per_warp(529) == 4 and lib.dm_streams_per_warp(6144) == 16 and lib.dm_streams_per_warp(4225) == 16


def test_bench_rank_partition_is_disjoint_and_complete():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    for world in (2, 4, 8):
        sets = [bench._my_blob_indices(64, r, world) for r in range(world)]
        assert all(len(s_) == 64 for s_ in sets)                       # weak scaling: same work per rank
        flat = [i for s_ in sets for i in s_]
        assert len(set(flat)) == len(flat)                             # no blob is hashed by two ranks
        top = max(flat)
        owners = {i: r for r, s_ in enumerate(sets) for i in s_}
        from demodel_b200.shard import owner_of_url
        assert all(owner_of_url(f"synthetic://blob/{i}", world) == r for i, r in owners.items())
        assert top < 64 * world * 3
    assert bench._my_blob_indices(5, 0, 1) == [0, 1, 2, 3, 4]
    assert bench._layout([1, 256, 257])[0] == [0, 256, 512] and bench._layout([1, 256, 257])[1] == 1024
