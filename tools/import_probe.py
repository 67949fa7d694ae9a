#!/usr/bin/env python3
"""How fast dm_cache_import seeds the disk tier from files already on the host.

Four shapes, one at a time: 4096 x 1 MiB, 256 x 16 MiB, 3000 files of 1..8192 bytes and 1 x 1 GiB.  Each shape's files
are written to a source directory, their SHA-256 taken with hashlib, and then imported twice with their digests known,
each time into an empty cas_dir by a new engine with a 512 MiB arena and the default ring (256 x 1 MiB slabs, so at
most 64 disk-backed checks in flight): once by copy, once by hard link (DM_IMP_LINK).  Source and cas_dir are on the
same filesystem, /dev/shm when it has room, so the two modes differ by the copy alone.  Per call:
  seconds        wall time of the call (it returns when every file is in the tier or has failed)
  GBps           bytes_hashed / seconds
  launches, launches_wide, launches_deep, launches_group, kernel_ms, bytes_hashed, h2d_bytes, blobs_committed: stat
                 deltas.  Which launch counter moves says which S (streams per warp) the pump chose: deep S = 1,
                 group 1 < S < 32, wide S = 32
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: import_probe.py [out.json]        env: BASE (directory for sources and cas_dir, default /dev/shm if it has room)
"""
import hashlib
import json
import os
import shutil
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

import demodel_b200  # noqa: E402
from promote_probe import bodies, gpu_info  # noqa: E402

ARENA = 512 << 20
SHAPES = [("4096x1MiB", 4096, 1 << 20), ("256x16MiB", 256, 16 << 20), ("3000x<=8KiB", 3000, 0), ("1x1GiB", 1, 1 << 30)]
COUNTERS = ("kernel_launches", "launches_wide", "launches_deep", "launches_group", "kernel_ms", "bytes_hashed",
            "h2d_bytes", "blobs_committed", "hbm_cas_used")


def write_sources(src, n, size):
    paths, digs = [], []
    if size == 0:                                            # the tiny shape: 1..8192 bytes each
        rng = np.random.default_rng(n)
        sizes = rng.integers(1, 8193, n)
        host = rng.integers(0, 256, int(sizes.sum()), dtype=np.uint8)
        offsets = np.concatenate([[0], np.cumsum(sizes)])
    else:
        host, offsets = bodies(n, size)
    for i in range(n):
        b = host[int(offsets[i]):int(offsets[i + 1])]
        p = os.path.join(src, f"f{i:05d}")
        with open(p, "wb") as f:
            f.write(b.tobytes())
        paths.append(p)
        digs.append(hashlib.sha256(b).digest())
    return paths, digs


def timed_import(base, paths, digs, link):
    cas = tempfile.mkdtemp(prefix="dm_import_probe_cas_", dir=base)
    try:
        with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=cas) as eng:
            st0 = eng.stats()
            t0 = time.perf_counter()
            res = eng.import_files(paths, expect=digs, link=link)
            secs = time.perf_counter() - t0
            st = eng.stats()
        assert res == [(demodel_b200.DM_OK, d) for d in digs], sorted({s for s, _ in res})
    finally:
        shutil.rmtree(cas, ignore_errors=True)
    r = {k: round(st[k] - st0[k], 3) if k == "kernel_ms" else st[k] - st0[k] for k in COUNTERS}
    r.update(files=len(paths), seconds=round(secs, 3), GBps=round(r["bytes_hashed"] / secs / 1e9, 3))
    return r


def main():
    base = os.environ.get("BASE", "/dev/shm")
    need = 2 * max(n * (size or 8192) for _, n, size in SHAPES) + (1 << 30)
    if not os.path.isdir(base) or shutil.disk_usage(base).free < need:
        base = tempfile.gettempdir()
    res = {"gpu": gpu_info(), "arena_bytes": ARENA, "on": base, "shapes": {}}
    if shutil.disk_usage(base).free < need:
        res["skipped"] = "not enough free space"
        print(json.dumps(res))
        return
    for name, n, size in SHAPES:
        src = tempfile.mkdtemp(prefix="dm_import_probe_src_", dir=base)
        try:
            paths, digs = write_sources(src, n, size)
            res["shapes"][name] = {mode: timed_import(base, paths, digs, mode == "link") for mode in ("copy", "link")}
            print(name, json.dumps(res["shapes"][name]), flush=True)
        finally:
            shutil.rmtree(src, ignore_errors=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
