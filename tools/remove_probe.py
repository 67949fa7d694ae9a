#!/usr/bin/env python3
"""What dm_cache_remove costs, with the cas_dir on /dev/shm (tmpfs).

  bulk      10 000 distinct 4 KiB blobs, cached through ordinary streams and made disk-only by an engine restart, removed
            by ONE dm_cache_remove call: its wall time, without a disk-tier limit and with one set (the limit index is
            built before the timed call).  Twice each, for the spread.
  opens     dm_cache_open + dm_cache_close latency of blobs that stay cached (256 in HBM, 256 on the disk tier only),
            alone and while another thread removes 10 000 other disk-only blobs in calls of 100: p50 and p99 of each.
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: remove_probe.py [out.json]       env: BASE (directory for the cas_dir, default /dev/shm)
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

ARENA = 1 << 30
N, SIZE, KEEP = 10_000, 4096, 256


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as ex:                         # reported, not fatal: the numbers then lack their context
        return {"error": str(ex)}


def populate(root, n, seed):
    """n distinct SIZE-byte blobs cached under root, disk-only once the engine is gone; returns their digests."""
    host = np.random.default_rng(seed).integers(0, 256, n * SIZE, dtype=np.uint8)
    offsets = np.arange(n + 1, dtype=np.uint64) * SIZE
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
        digs, ok, _ = eng.proxy_drive(host, offsets, chunk=SIZE, concurrency=256, nthreads=8)
        assert all(ok)
    return digs


def pct(xs, p):
    return float(np.percentile(np.asarray(xs) * 1e6, p))


def bulk(base, limit):
    root = tempfile.mkdtemp(dir=base, prefix="dm_rm_probe_")
    try:
        digs = populate(root, N, 1 + limit)
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
            if limit:
                eng.set_disk_limit(1 << 40)
            t = time.perf_counter()
            st = eng.cache_remove(digs)
            dt = time.perf_counter() - t
            assert st == [demodel_b200.DM_OK] * N and not eng.list(cap=1)
        return dt
    finally:
        shutil.rmtree(root, ignore_errors=True)


def opens(base):
    root = tempfile.mkdtemp(dir=base, prefix="dm_rm_probe_")
    try:
        victims = populate(root, N, 7)
        cold = populate(root, KEEP, 8)
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=root) as eng:
            hot = [eng.ingest(np.random.default_rng(9 + i).integers(0, 256, SIZE, dtype=np.uint8))[0] for i in range(KEEP)]

            def sample(digs, rounds):
                lat = []
                for _ in range(rounds):
                    for d in digs:
                        t = time.perf_counter()
                        rid, _ = eng.cache_open(d)
                        eng.cache_close(rid)
                        lat.append(time.perf_counter() - t)
                return lat
            out = {}
            for name, digs in (("hbm", hot), ("disk", cold)):
                sample(digs, 1)
                out[f"{name}_alone"] = sample(digs, 8)
            done = threading.Event()
            removed = []

            def remover():
                t = time.perf_counter()
                for i in range(0, N, 100):
                    removed.extend(eng.cache_remove(victims[i:i + 100]))
                removed.append(time.perf_counter() - t)
                done.set()
            th = threading.Thread(target=remover)
            th.start()
            during = {"hbm": [], "disk": []}
            while not done.is_set():
                for name, digs in (("hbm", hot), ("disk", cold)):
                    during[name] += sample(digs[:64], 1)
            th.join()
            remove_s = removed.pop()
            assert removed == [demodel_b200.DM_OK] * N
        res = {"remove_10k_in_calls_of_100_s": remove_s}
        for name in ("hbm", "disk"):
            res[f"open_{name}_alone_p50_us"] = pct(out[f"{name}_alone"], 50)
            res[f"open_{name}_alone_p99_us"] = pct(out[f"{name}_alone"], 99)
            res[f"open_{name}_during_p50_us"] = pct(during[name], 50)
            res[f"open_{name}_during_p99_us"] = pct(during[name], 99)
            res[f"open_{name}_during_samples"] = len(during[name])
        return res
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "cas_base": base, "blobs": N, "blob_bytes": SIZE}
    res["remove_10k_no_limit_s"] = [bulk(base, 0) for _ in range(2)]
    res["remove_10k_with_limit_s"] = [bulk(base, 1) for _ in range(2)]
    res.update(opens(base))
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
