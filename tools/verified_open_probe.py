#!/usr/bin/env python3
"""What a verified hit (dm_cache_open_verified) costs against a plain disk-tier hit (dm_cache_open).

Every blob is cached through ordinary streams into a cas_dir on /dev/shm, and the engine is restarted over it, so that
each is on the disk tier only.
  single         a 64 MiB and a 1 GiB blob, read front to back by one reader (the first read 32 KiB, then 1 MiB
                 pieces): time to first byte and to last byte from the open, and to the EOF read.  Plain open first
                 (a pread of the file), then verified (the blob is loaded and hashed; the last byte waits for the
                 verdict), then the blob is evicted from HBM again; twice, for the spread.
  aggregate      256 distinct 4 MiB blobs opened verified at once from one thread, then read to EOF by 16 Python
                 threads in 1 MiB pieces: wall time from the first open to the last EOF, and GB/s.  The same with plain
                 opens after every blob was evicted from HBM again.  The readers are ctypes calls: each releases the GIL
                 while it runs but holds it between calls, so the plain figure is bound by the Python readers.
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: verified_open_probe.py [out.json]       env: BASE (directory for the cas_dir, default /dev/shm)
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import demodel_b200  # noqa: E402

ARENA = 8 << 30
SINGLE = [64 << 20, 1 << 30]
AGG_N, AGG_SIZE, AGG_THREADS = 256, 4 << 20, 16
FIRST, PIECE = 32 << 10, 1 << 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as ex:                         # reported, not fatal: the numbers then lack their context
        return {"error": str(ex)}


def bodies(n, size):
    """n distinct bodies of `size` bytes in one host array: a random pool, each body stamped with its index."""
    pool = np.random.default_rng(n * 7 + size).integers(0, 256, min(size, 64 << 20), dtype=np.uint8)
    host = np.tile(pool, (n * size + pool.nbytes - 1) // pool.nbytes)[:n * size]
    stamps = host.reshape(n, size)[:, :8]
    stamps[:] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
    return host, np.arange(n + 1, dtype=np.uint64) * size


def populate(root, n, size):
    host, offsets = bodies(n, size)
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
        digs, ok, _ = eng.proxy_drive(host, offsets, chunk=1 << 20, concurrency=min(n, 256), nthreads=8)
        assert all(ok)
    return digs


def read_through(eng, rid, size, t0):
    """Read to EOF: (first byte, last byte, EOF) seconds after t0."""
    first = last = None
    off = 0
    while off < size:
        part = eng.cache_read(rid, off, FIRST if off == 0 else PIECE)
        assert part
        off += len(part)
        now = time.perf_counter()
        if first is None:
            first = now - t0
        if off == size:
            last = now - t0
    assert eng.cache_read(rid, size, PIECE) == b""
    return first, last, time.perf_counter() - t0


def single(base, size):
    root = tempfile.mkdtemp(prefix="dm_verified_probe_", dir=base)
    try:
        (dig,) = populate(root, 1, size)
        runs = []
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:    # restart: disk tier only
            for _ in range(2):
                for kind, opener in (("plain", eng.cache_open), ("verified", eng.cache_open_verified)):
                    st0 = eng.stats()
                    t0 = time.perf_counter()
                    rid, n = opener(dig)
                    opened = time.perf_counter() - t0
                    first, last, eof = read_through(eng, rid, n, t0)
                    eng.cache_close(rid)
                    st = eng.stats()
                    runs.append({"open": kind, "open_s": round(opened, 6), "first_byte_s": round(first, 6),
                                 "last_byte_s": round(last, 4), "eof_s": round(eof, 4),
                                 "bytes_hashed": st["bytes_hashed"] - st0["bytes_hashed"]})
                assert eng.cache_evict(dig)
        return {"blob_bytes": size, "runs": runs}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def aggregate(base):
    root = tempfile.mkdtemp(prefix="dm_verified_probe_", dir=base)
    try:
        digs = populate(root, AGG_N, AGG_SIZE)
        runs = []
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
            for kind, opener in (("verified", eng.cache_open_verified), ("plain", eng.cache_open)):
                st0 = eng.stats()
                t0 = time.perf_counter()
                opened = [opener(d) for d in digs]
                open_s = time.perf_counter() - t0
                todo = list(opened)
                lock = threading.Lock()

                def reader():
                    while True:
                        with lock:
                            if not todo:
                                return
                            rid, n = todo.pop()
                        off = 0
                        while off < n:
                            off += len(eng.cache_read(rid, off, PIECE))
                        assert eng.cache_read(rid, n, PIECE) == b""
                        eng.cache_close(rid)
                th = [threading.Thread(target=reader) for _ in range(AGG_THREADS)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                secs = time.perf_counter() - t0
                st = eng.stats()
                runs.append({"open": kind, "opens_s": round(open_s, 4), "seconds": round(secs, 4),
                             "GBps": round(AGG_N * AGG_SIZE / secs / 1e9, 3),
                             "bytes_hashed": st["bytes_hashed"] - st0["bytes_hashed"],
                             "kernel_launches": st["kernel_launches"] - st0["kernel_launches"]})
                for d in digs:
                    eng.cache_evict(d)
        return {"blobs": AGG_N, "blob_bytes": AGG_SIZE, "reader_threads": AGG_THREADS, "runs": runs}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "arena_bytes": ARENA, "cas_dir_on": base, "single": [], "aggregate": None}
    for size in SINGLE:
        r = single(base, size)
        res["single"].append(r)
        print(json.dumps(r), flush=True)
    res["aggregate"] = aggregate(base)
    print(json.dumps(res["aggregate"]), flush=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
