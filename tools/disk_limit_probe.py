#!/usr/bin/env python3
"""What the disk-tier limit (dm_cache_set_disk_limit) costs.

Three measurements, each on a fresh cas_dir under BASE:
  walk            seconds of the first dm_cache_set_disk_limit over 20 000 and 100 000 blob files (1 byte each, with a
                  sidecar): the one walk that builds the index, a stat per name
  spill           256 x 16 MiB through 32 concurrent streams into an HBM engine (DM_F_DISK_SYNC, so dm_stream_finish
                  returns once the spill is on disk), with no limit and with a limit that holds 64 of them: wall seconds,
                  GB/s (bytes / seconds, hash and spill together) and p50 / p99 of dm_stream_finish
  open_read       p50 / p99 of dm_cache_open + a 4 KiB dm_cache_read + dm_cache_close of random disk-only blobs (512 x
                  64 KiB), with no limit and with one: the cost of writing the mtime of each opened file
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: disk_limit_probe.py [out.json]     env: BASE (directories for the cas_dirs, comma-separated, default /dev/shm),
                                               WALK=0 skips the walk
"""
import json
import os
import shutil
import sys
import tempfile
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

import demodel_b200  # noqa: E402
from demodel_b200._lib import DM_F_DISK_SYNC  # noqa: E402
from promote_probe import bodies, gpu_info  # noqa: E402

SPILL_N, SPILL_SIZE, SPILL_HOLD, SPILL_STREAMS = 256, 16 << 20, 64, 32
OPEN_N, OPEN_SIZE, OPEN_READS = 512, 64 << 10, 4000


def pct(xs, q):
    return round(float(np.percentile(np.asarray(xs) * 1e6, q)), 1)


def walk(base, n):
    cas = tempfile.mkdtemp(prefix="dm_limit_probe_walk_", dir=base)
    try:
        rng = np.random.default_rng(n)
        for i in range(n):
            hx = rng.bytes(32).hex()
            d = os.path.join(cas, "blobs", "sha256", hx[:2])
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, hx), "wb") as f:
                f.write(b"x")
            with open(os.path.join(d, hx + ".meta"), "w") as f:
                f.write("{}\n")
        with demodel_b200.Engine(device=0, hbm_cas_bytes=64 << 20, cas_dir=cas) as eng:
            t0 = time.perf_counter()
            eng.set_disk_limit(1 << 60)
            secs = time.perf_counter() - t0
            u = eng.disk_usage()
        assert u["blob_files"] == n, u
        return {"files": n, "seconds": round(secs, 4)}
    finally:
        shutil.rmtree(cas, ignore_errors=True)


def spill(base, limit, host):
    cas = tempfile.mkdtemp(prefix="dm_limit_probe_spill_", dir=base)
    try:
        with demodel_b200.Engine(device=0, hbm_cas_bytes=SPILL_N * SPILL_SIZE + (256 << 20), cas_dir=cas,
                                 flags=DM_F_DISK_SYNC) as eng:
            if limit:
                eng.set_disk_limit(SPILL_HOLD * (SPILL_SIZE + 512))
            fin = []

            def writer(k):                             # SPILL_STREAMS bodies in flight, so the hash is not one chain
                for i in range(k, SPILL_N, SPILL_STREAMS):
                    body = host[i * SPILL_SIZE:(i + 1) * SPILL_SIZE]
                    sid = eng.stream_open(None, SPILL_SIZE)
                    for off in range(0, SPILL_SIZE, 1 << 20):
                        eng.stream_write(sid, body[off:off + (1 << 20)])
                    t1 = time.perf_counter()
                    _, ok = eng.stream_finish(sid)
                    fin.append(time.perf_counter() - t1)
                    assert ok

            t0 = time.perf_counter()
            th = [threading.Thread(target=writer, args=(k,)) for k in range(SPILL_STREAMS)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert len(fin) == SPILL_N
            secs = time.perf_counter() - t0
            u = eng.disk_usage()
        return {"limit": bool(limit), "seconds": round(secs, 3), "spill_GBps": round(SPILL_N * SPILL_SIZE / secs / 1e9, 3),
                "finish_p50_us": pct(fin, 50), "finish_p99_us": pct(fin, 99), "evicted_files": u["evicted_files"]}
    finally:
        shutil.rmtree(cas, ignore_errors=True)


def open_read(base, limit):
    cas = tempfile.mkdtemp(prefix="dm_limit_probe_open_", dir=base)
    rng = np.random.default_rng(11)
    try:
        with demodel_b200.Engine(device=0, hbm_cas_bytes=256 << 20, cas_dir=cas, flags=DM_F_DISK_SYNC) as eng:
            if limit:
                eng.set_disk_limit(1 << 50)
            digs = []
            for i in range(OPEN_N):
                body = rng.integers(0, 256, OPEN_SIZE, dtype=np.uint8)
                sid = eng.stream_open(None, OPEN_SIZE)
                eng.stream_write(sid, body)
                d, ok = eng.stream_finish(sid)
                assert ok and eng.cache_evict(d)
                digs.append(d)
            lat = []
            for k in rng.integers(0, OPEN_N, OPEN_READS):
                t0 = time.perf_counter()
                rid, _ = eng.cache_open(digs[k])
                eng.cache_read(rid, 0, 4096)
                eng.cache_close(rid)
                lat.append(time.perf_counter() - t0)
        return {"limit": bool(limit), "reads": OPEN_READS, "p50_us": pct(lat, 50), "p99_us": pct(lat, 99)}
    finally:
        shutil.rmtree(cas, ignore_errors=True)


def main():
    bases = [b for b in os.environ.get("BASE", "/dev/shm").split(",") if b]
    res = {"gpu": gpu_info(), "runs": {}}
    need = SPILL_N * SPILL_SIZE + (1 << 30)
    for base in bases:
        if not os.path.isdir(base) or shutil.disk_usage(base).free < need:
            res["runs"][base] = {"skipped": "not enough free space"}
            continue
        r = res["runs"][base] = {"walk": [], "spill": [], "open_read": []}
        for n in ((20000, 100000) if os.environ.get("WALK", "1") == "1" else ()):
            r["walk"].append(walk(base, n))
            print(base, "walk", r["walk"][-1], flush=True)
        host, _ = bodies(SPILL_N, SPILL_SIZE)
        for lim in (False, True):
            r["spill"].append(spill(base, lim, host))
            print(base, "spill", r["spill"][-1], flush=True)
        del host
        for lim in (False, True, False, True):
            r["open_read"].append(open_read(base, lim))
            print(base, "open_read", r["open_read"][-1], flush=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
