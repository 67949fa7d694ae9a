"""TEST INFRASTRUCTURE: host-side cost of dm_ingest_device per blob for 10^5-blob batches, measured on the CPU box
against the fake runtime with its kernels switched off (FAKE_CUDA_NULL_KERNEL=2: "digests" are a mix of the source
address, nothing is copied or verified).  What remains is what the GPU box spends on the host around the launch: extents,
job table, eviction of the previous copies, verification, publication.
usage: bulk_cost_probe.py <fake libdemodel_b200.so> [n] [steps]"""
import os
import sys
import time

os.environ["FAKE_CUDA_NULL_KERNEL"] = "2"
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import demodel_b200._lib as _lib  # noqa: E402

_lib.LIB_PATH = sys.argv[1]
import numpy as np  # noqa: E402
import demodel_b200  # noqa: E402

n = int(sys.argv[2]) if len(sys.argv) > 2 else 135168
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
size = 256
host = np.zeros(n * size, dtype=np.uint8)             # "device" memory of the fake runtime is host memory
off = np.arange(n, dtype=np.uint64) * np.uint64(size)
ln = np.full(n, size, dtype=np.uint64)
with demodel_b200.Engine(device=0, hbm_cas_bytes=(n * size * 2) + (64 << 20), ring_bytes=16 << 20, max_streams=4096) as eng:
    d, _, _ = eng.ingest_device(host.ctypes.data, off, ln, hash_only=True, raw=True)
    expect = d.tobytes()
    assert len(set(expect[32 * i:32 * i + 32] for i in range(0, n, 97))) == len(range(0, n, 97))
    for phase in ("hash-only", "hash + cache, replacing the previous copies"):
        ts = []
        for _ in range(steps + 2):
            t0 = time.perf_counter()
            d, m, _ = eng.ingest_device(host.ctypes.data, off, ln, expect=expect, hash_only=phase == "hash-only", replace=True, raw=True)
            ts.append(time.perf_counter() - t0)
            assert m.all()
        best = min(ts[2:])
        print(f"{phase}: {n} blobs, best of {steps}: {best * 1e3:7.2f} ms per call = {best / n * 1e9:6.1f} ns per blob"
              f"  (first call, everything new: {ts[0] * 1e3:.2f} ms)")
    st = eng.stats()
    print(f"launches: {st['kernel_launches']} ({st['launches_wide']} lane-per-stream), blobs committed: {st['blobs_committed']}")
