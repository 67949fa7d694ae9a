#!/usr/bin/env python3
"""What sharing one ring load among the Range: readers of a blob saves (dm_cache_open_verified_range against
dm_cache_open_verified_ring).

A 1 GiB blob is cached through an ordinary stream into a cas_dir on /dev/shm, and the serving engine has an arena smaller
than the blob, so every hit on it is served from the disk tier through ring slabs.  The blob is then fetched as N equal
parts (N = 1, 4, 16), each part opened and read concurrently by a Python thread of its own in 1 MiB pieces, the way a
parallel downloader's Range: requests arrive at a proxy:
  ring    each part a ring open (dm_cache_open_verified_ring) whose first read is at the part's offset
  range   each part a range open (dm_cache_open_verified_range) of the part's bytes
For each, twice: the wall time from the first open to the last part's end, the time to each part's last byte,
bytes_hashed and h2d_bytes, and how many opens were refused (DM_ENOMEM).  The engine's ring is RING bytes of 1 MiB slabs:
ring loads may hold a quarter of them, 4 slabs each.  The GPU's name, power limit and SM clocks are read (nvidia-smi
--query-gpu, read-only) in the same run.

usage: verified_range_probe.py [out.json]       env: BASE (directory for the cas_dir, default /dev/shm)
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

SIZE = 1 << 30
PARTS = [1, 4, 16]
RING = 128 << 20            # 128 slabs of 1 MiB: ring loads may hold 32, i.e. 8 ring loads at once
PIECE = 1 << 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as ex:                         # reported, not fatal: the numbers then lack their context
        return {"error": str(ex)}


def populate(root):
    body = np.random.default_rng(7).integers(0, 256, SIZE, dtype=np.uint8)
    with demodel_b200.Engine(device=0, hbm_cas_bytes=2 << 30, cas_dir=root) as eng:
        digs, ok, _ = eng.proxy_drive(body, np.array([0, SIZE], dtype=np.uint64), chunk=1 << 20, concurrency=1,
                                      nthreads=1)
    assert all(ok)
    return digs[0]


def fetch(eng, dig, n, kind):
    step = SIZE // n
    parts = [(k * step, step if k < n - 1 else SIZE - k * step) for k in range(n)]
    st0 = eng.stats()
    t0 = time.perf_counter()
    done, refused = [None] * n, [0]

    def part(k):
        off, ln = parts[k]
        try:
            rid, size = (eng.cache_open_verified_ring(dig) if kind == "ring"
                         else eng.cache_open_verified_range(dig, off, ln))
        except demodel_b200.DmError as ex:
            assert ex.code == demodel_b200.DM_ENOMEM
            refused[0] += 1
            return
        try:
            pos = off
            while pos < off + ln:
                got = eng.cache_read(rid, pos, min(PIECE, off + ln - pos))
                assert got
                pos += len(got)
            done[k] = time.perf_counter() - t0
        finally:
            eng.cache_close(rid)
    th = [threading.Thread(target=part, args=(k,)) for k in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    wall = time.perf_counter() - t0
    st = eng.stats()
    served = [d for d in done if d is not None]
    return {"kind": kind, "parts": n, "served": len(served), "refused_enomem": refused[0], "wall_s": wall,
            "part_last_byte_s": [round(d, 3) if d is not None else None for d in done],
            "bytes_hashed": st["bytes_hashed"] - st0["bytes_hashed"], "h2d_bytes": st["h2d_bytes"] - st0["h2d_bytes"]}


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "cas_dir_on": base, "blob_bytes": SIZE, "ring_bytes": RING, "runs": []}
    root = tempfile.mkdtemp(prefix="dm_range_probe_", dir=base)
    try:
        dig = populate(root)
        with demodel_b200.Engine(device=0, hbm_cas_bytes=256 << 20, ring_bytes=RING, slab_bytes=1 << 20,
                                 cas_dir=root) as eng:
            for _ in range(2):
                for n in PARTS:
                    for kind in ("ring", "range"):
                        r = fetch(eng, dig, n, kind)
                        res["runs"].append(r)
                        print(json.dumps(r), flush=True)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
