#!/usr/bin/env python3
"""How fast dm_cache_verify checks disk-tier files in place on the GPU.

One cas_dir is populated with four shapes: 4096 x 1 MiB, 256 x 16 MiB and 3000 bodies of 1..8192 bytes through ordinary
streams (dm_proxy_drive), and 1 x 1 GiB through a disk-backed stream on an engine whose arena (512 MiB) is smaller than
it.  Then a new engine is created over the directory, with the same 512 MiB arena and the default ring (256 x 1 MiB
slabs, so at most 64 disk-backed checks in flight), and one dm_cache_verify call over every blob is timed, twice (the
spread of the two is the spread of the number).  Then one call per shape is timed.  Per call:
  seconds        wall time of the call (it returns when every file has its verdict)
  GBps           bytes_hashed / seconds
  launches, launches_wide, launches_deep, launches_group, kernel_ms, bytes_hashed, h2d_bytes: stat deltas.  Which
                 launch counter moves says which S (streams per warp) the pump chose: deep S = 1, group 1 < S < 32,
                 wide S = 32
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: verify_probe.py [out.json]        env: BASE (directory for the cas_dir, default /dev/shm if it has room)
"""
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
from demodel_b200._lib import DM_F_DISK_DIRECT  # noqa: E402
from promote_probe import bodies, gpu_info  # noqa: E402

POPULATE_ARENA = 8 << 30
VERIFY_ARENA = 512 << 20
SHAPES = [("4096x1MiB", 4096, 1 << 20), ("256x16MiB", 256, 16 << 20)]
TINY = 3000
HUGE = 1 << 30
COUNTERS = ("kernel_launches", "launches_wide", "launches_deep", "launches_group", "kernel_ms", "bytes_hashed",
            "h2d_bytes", "hbm_cas_used")


def timed_verify(eng, digs):
    st0 = eng.stats()
    t0 = time.perf_counter()
    status = eng.verify(digs)
    secs = time.perf_counter() - t0
    st = eng.stats()
    assert status == [demodel_b200.DM_OK] * len(digs), sorted(set(status))
    r = {k: round(st[k] - st0[k], 3) if k == "kernel_ms" else st[k] - st0[k] for k in COUNTERS}
    r.update(blobs=len(digs), seconds=round(secs, 3), GBps=round(r["bytes_hashed"] / secs / 1e9, 3))
    return r


def populate(root):
    digs = {}
    for name, n, size in SHAPES:
        host, offsets = bodies(n, size)
        with demodel_b200.Engine(device=0, hbm_cas_bytes=POPULATE_ARENA, cas_dir=root) as eng:
            d, ok, _ = eng.proxy_drive(host, offsets, chunk=1 << 20, concurrency=min(n, 256), nthreads=8)
            assert all(ok)
        digs[name] = d
        del host
    rng = np.random.default_rng(TINY)
    sizes = rng.integers(1, 8193, TINY)
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    host = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    with demodel_b200.Engine(device=0, hbm_cas_bytes=POPULATE_ARENA, cas_dir=root) as eng:
        d, ok, _ = eng.proxy_drive(host, offsets, concurrency=64, nthreads=4)
        assert all(ok)
    digs[f"{TINY}x<=8KiB"] = d
    huge = np.random.default_rng(HUGE).integers(0, 256, HUGE, dtype=np.uint8)
    with demodel_b200.Engine(device=0, hbm_cas_bytes=VERIFY_ARENA, cas_dir=root, flags=DM_F_DISK_DIRECT) as eng:
        sid = eng.stream_open(None, HUGE)                    # larger than the arena: a disk-backed stream
        for off in range(0, HUGE, 1 << 20):
            eng.stream_write(sid, huge[off:off + (1 << 20)])
        d, ok = eng.stream_finish(sid)
        assert ok
    digs["1x1GiB"] = [d]
    return digs


def main():
    base = os.environ.get("BASE", "/dev/shm")
    need = sum(n * size for _, n, size in SHAPES) + TINY * 8192 + HUGE + (1 << 30)
    if shutil.disk_usage(base).free < need:
        base = tempfile.gettempdir()
    res = {"gpu": gpu_info(), "verify_arena_bytes": VERIFY_ARENA, "cas_dir_on": base}
    if shutil.disk_usage(base).free < need:
        res["skipped"] = "not enough free space"
        print(json.dumps(res))
        return
    root = tempfile.mkdtemp(prefix="dm_verify_probe_", dir=base)
    try:
        digs = populate(root)
        everything = [d for v in digs.values() for d in v]
        with demodel_b200.Engine(device=0, hbm_cas_bytes=VERIFY_ARENA, cas_dir=root) as eng:    # restart
            res["ring_slabs"] = eng.stats()["ring_slabs_total"]
            res["all"] = [timed_verify(eng, everything) for _ in range(2)]
            print(json.dumps(res["all"]), flush=True)
            res["shapes"] = {name: timed_verify(eng, d) for name, d in digs.items()}
            print(json.dumps(res["shapes"]), flush=True)
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
