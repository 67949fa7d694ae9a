#!/usr/bin/env python3
"""What a ring-load hit (dm_cache_open_verified_ring) costs, on an engine without an HBM tier (DM_F_NO_HBM_CAS).

Every blob is cached through ordinary streams into a cas_dir on /dev/shm, and the serving engine has no HBM tier, so each
is on the disk tier only and every hit is a ring load.
  single         a 64 MiB and a 1 GiB blob, read front to back by one reader (the first read 32 KiB, then 1 MiB
                 pieces): the open's own latency, and the time from the open to the first byte, to the last byte (it
                 waits for the verdict) and to the EOF read; twice, for the spread.  The same blob opened plainly
                 (dm_cache_open, an unverified pread of the file) is the reference.
  aggregate      256 distinct 4 MiB blobs opened through ring loads at once from one thread, on a ring large enough that
                 the ring-load share admits all of them, then read to EOF by 16 Python threads in 1 MiB pieces: wall
                 time from the first open to the last EOF, GB/s, and how many opens were refused (DM_ENOMEM).
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: verified_ring_probe.py [out.json]       env: BASE (directory for the cas_dir, default /dev/shm)
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
from demodel_b200._lib import DM_F_NO_HBM_CAS  # noqa: E402

SINGLE = [64 << 20, 1 << 30]
AGG_N, AGG_SIZE, AGG_THREADS = 256, 4 << 20, 16
AGG_RING = 4 << 30          # 4096 slabs of 1 MiB: a quarter of them is 256 loads of 4 slabs
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
    with demodel_b200.Engine(device=0, hbm_cas_bytes=8 << 30, cas_dir=root) as eng:
        digs, ok, _ = eng.proxy_drive(host, offsets, chunk=1 << 20, concurrency=min(n, 256), nthreads=8)
    assert all(ok)
    return digs, host


def read_timed(eng, rid, size, t0):
    first = last = None
    off = 0
    while off < size:
        part = eng.cache_read(rid, off, FIRST if off == 0 else PIECE)
        assert part
        if first is None:
            first = time.perf_counter() - t0
        off += len(part)
        if off == size:
            last = time.perf_counter() - t0
    assert eng.cache_read(rid, size, PIECE) == b""
    return first, last, time.perf_counter() - t0


def single(base, size):
    root = tempfile.mkdtemp(prefix="dm_ring_probe_", dir=base)
    try:
        (dig,), _ = populate(root, 1, size)
        runs = []
        with demodel_b200.Engine(device=0, hbm_cas_bytes=1 << 30, flags=DM_F_NO_HBM_CAS, cas_dir=root) as eng:
            for _ in range(2):
                for kind, opener in (("plain", eng.cache_open), ("ring", eng.cache_open_verified_ring)):
                    st0 = eng.stats()
                    t0 = time.perf_counter()
                    rid, got = opener(dig)
                    t_open = time.perf_counter() - t0
                    first, last, eof = read_timed(eng, rid, got, t0)
                    eng.cache_close(rid)
                    st = eng.stats()
                    runs.append({"kind": kind, "open_ms": t_open * 1e3, "first_byte_ms": first * 1e3,
                                 "last_byte_s": last, "eof_s": eof, "MB_per_s_to_eof": size / eof / 1e6,
                                 "bytes_hashed": st["bytes_hashed"] - st0["bytes_hashed"],
                                 "hbm_cas_used": st["hbm_cas_used"]})
        return {"size": size, "runs": runs}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def aggregate(base):
    root = tempfile.mkdtemp(prefix="dm_ring_probe_", dir=base)
    try:
        digs, _ = populate(root, AGG_N, AGG_SIZE)
        runs = []
        with demodel_b200.Engine(device=0, hbm_cas_bytes=1 << 30, flags=DM_F_NO_HBM_CAS, ring_bytes=AGG_RING,
                                 cas_dir=root) as eng:
            for _ in range(2):
                st0 = eng.stats()
                t0 = time.perf_counter()
                opened, refused = [], 0
                for d in digs:
                    try:
                        opened.append(eng.cache_open_verified_ring(d))
                    except demodel_b200.DmError as ex:
                        assert ex.code == demodel_b200.DM_ENOMEM
                        refused += 1
                t_open = time.perf_counter() - t0
                todo = list(opened)
                lock = threading.Lock()

                def worker():
                    while True:
                        with lock:
                            if not todo:
                                return
                            rid, size = todo.pop()
                        off = 0
                        while off < size:
                            part = eng.cache_read(rid, off, PIECE)
                            assert part
                            off += len(part)
                        assert eng.cache_read(rid, size, PIECE) == b""
                        eng.cache_close(rid)
                th = [threading.Thread(target=worker) for _ in range(AGG_THREADS)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                wall = time.perf_counter() - t0
                st = eng.stats()
                runs.append({"opened": len(opened), "refused_enomem": refused, "open_all_ms": t_open * 1e3,
                             "wall_s": wall, "GB_per_s": len(opened) * AGG_SIZE / wall / 1e9,
                             "bytes_hashed": st["bytes_hashed"] - st0["bytes_hashed"],
                             "kernel_launches": st["kernel_launches"] - st0["kernel_launches"],
                             "ring_slabs_free_after": st["ring_slabs_free"], "ring_slabs_total": st["ring_slabs_total"]})
        return {"blobs": AGG_N, "blob_bytes": AGG_SIZE, "reader_threads": AGG_THREADS, "ring_bytes": AGG_RING,
                "runs": runs}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "cas_dir_on": base, "single": [], "aggregate": None}
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
