#!/usr/bin/env python3
"""How fast dm_cache_promote brings disk-tier blobs back into HBM, verifying each on the GPU as it loads.

For each shape (4096 x 1 MiB, 256 x 16 MiB, 1 x 1 GiB) a cas_dir on /dev/shm is populated through ordinary streams
(dm_proxy_drive), the engine is destroyed and a new one is created over the same directory, so that every blob is on
the disk tier only.  Then one dm_cache_promote call over all of them is timed; every blob is evicted again and the
call is timed a second time (the spread of the two is the spread of the number).  Per call:
  seconds        wall time of the call (it returns when every blob is hashed and published)
  GBps           bytes / seconds
  launches, launches_wide, launches_deep, launches_group, kernel_ms, bytes_hashed, h2d_bytes: stat deltas
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: promote_probe.py [out.json]       env: BASE (directory for the cas_dir, default /dev/shm)
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import demodel_b200  # noqa: E402

ARENA = 8 << 30
SHAPES = [(4096, 1 << 20), (256, 16 << 20), (1, 1 << 30)]
COUNTERS = ("kernel_launches", "launches_wide", "launches_deep", "launches_group", "kernel_ms", "bytes_hashed",
            "h2d_bytes")


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
    pool = np.random.default_rng(n).integers(0, 256, min(size, 64 << 20), dtype=np.uint8)
    host = np.tile(pool, (n * size + pool.nbytes - 1) // pool.nbytes)[:n * size]
    stamps = host.reshape(n, size)[:, :8]
    stamps[:] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
    return host, np.arange(n + 1, dtype=np.uint64) * size


def timed_promote(eng, digs):
    st0 = eng.stats()
    t0 = time.perf_counter()
    status = eng.promote(digs)
    secs = time.perf_counter() - t0
    st = eng.stats()
    assert status == [demodel_b200.DM_OK] * len(digs), sorted(set(status))
    r = {k: round(st[k] - st0[k], 3) if k == "kernel_ms" else st[k] - st0[k] for k in COUNTERS}
    r.update(seconds=round(secs, 3), GBps=round(r["bytes_hashed"] / secs / 1e9, 3))
    return r


def one_shape(base, n, size):
    root = tempfile.mkdtemp(prefix="dm_promote_probe_", dir=base)
    try:
        host, offsets = bodies(n, size)
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
            digs, ok, _ = eng.proxy_drive(host, offsets, chunk=1 << 20, concurrency=min(n, 256), nthreads=8)
            assert all(ok)
        del host
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:    # restart: disk tier only
            runs = [timed_promote(eng, digs)]
            for d in digs:
                eng.cache_evict(d)
            runs.append(timed_promote(eng, digs))
        return {"blobs": n, "blob_bytes": size, "runs": runs}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "arena_bytes": ARENA, "cas_dir_on": base, "shapes": []}
    for n, size in SHAPES:
        if shutil.disk_usage(base).free < n * size + (1 << 30):
            res["shapes"].append({"blobs": n, "blob_bytes": size, "skipped": "not enough free space"})
            continue
        r = one_shape(base, n, size)
        res["shapes"].append(r)
        print(json.dumps(r), flush=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
