#!/usr/bin/env python3
"""How fast dm_cache_export writes cached blobs out, each copy hashed on the GPU before it is renamed into place.

Four shapes, one at a time: 4096 x 1 MiB, 256 x 16 MiB, 3000 files of 1..8192 bytes and 1 x 1 GiB.  Each shape's
files are written to a source directory, their SHA-256 taken with hashlib, and imported into an empty cas_dir.  A new
engine (6 GiB arena, the default ring: 256 x 1 MiB slabs, of which an export may hold a quarter) then exports them
twice into empty directories:
  disk           every blob on the disk tier only (copy_file_range into the staged file, read back through the ring)
  hbm            after dm_cache_promote put every blob in HBM as well (D2H into the staged file, read back the same way)
cas_dir and destinations are on /dev/shm when it has room.  Per export:
  seconds        wall time of the call (it returns when every file is in place or has failed)
  GBps           bytes exported / seconds
  launches, kernel_ms, bytes_hashed, h2d_bytes, d2h_bytes, packed_bodies: stat deltas
The probe asserts that bytes_hashed grew by exactly the bytes exported and that every destination hashes to its digest
(a sample of 64 files per shape, read back with hashlib).  The GPU's name, power limit and SM clocks are read
(nvidia-smi --query-gpu, read-only) in the same run.

usage: export_probe.py [out.json]        env: BASE (directory for sources, cas_dir and destinations)
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

import demodel_b200  # noqa: E402
from import_probe import SHAPES, write_sources  # noqa: E402
from promote_probe import gpu_info  # noqa: E402

ARENA = 6 << 30
COUNTERS = ("kernel_launches", "kernel_ms", "bytes_hashed", "h2d_bytes", "d2h_bytes", "packed_bodies", "hbm_cas_used",
            "blobs_committed")


def timed_export(eng, base, digs, sizes):
    out = tempfile.mkdtemp(prefix="dm_export_probe_out_", dir=base)
    try:
        dests = [os.path.join(out, f"f{i:05d}") for i in range(len(digs))]
        st0 = eng.stats()
        t0 = time.perf_counter()
        res = eng.export(digs, dests)
        secs = time.perf_counter() - t0
        st = eng.stats()
        assert res == [demodel_b200.DM_OK] * len(digs), sorted(set(res))
        step = max(1, len(digs) // 64)
        for d, p in zip(digs[::step], dests[::step]):
            h = hashlib.sha256()
            with open(p, "rb") as f:
                for chunk in iter(lambda: f.read(1 << 24), b""):
                    h.update(chunk)
            assert h.digest() == d, p
    finally:
        shutil.rmtree(out, ignore_errors=True)
    r = {k: round(st[k] - st0[k], 3) if k == "kernel_ms" else st[k] - st0[k] for k in COUNTERS}
    assert r["bytes_hashed"] == sum(sizes), (r["bytes_hashed"], sum(sizes))
    assert r["hbm_cas_used"] == 0 and r["blobs_committed"] == 0
    r.update(files=len(digs), seconds=round(secs, 3), GBps=round(sum(sizes) / secs / 1e9, 3))
    return r


def main():
    base = os.environ.get("BASE", "/dev/shm")
    need = 3 * max(n * (size or 8192) for _, n, size in SHAPES) + (1 << 30)
    if not os.path.isdir(base) or shutil.disk_usage(base).free < need:
        base = tempfile.gettempdir()
    res = {"gpu": gpu_info(), "arena_bytes": ARENA, "on": base, "shapes": {}}
    if shutil.disk_usage(base).free < need:
        res["skipped"] = "not enough free space"
        print(json.dumps(res))
        return
    for name, n, size in SHAPES:
        src = tempfile.mkdtemp(prefix="dm_export_probe_src_", dir=base)
        cas = tempfile.mkdtemp(prefix="dm_export_probe_cas_", dir=base)
        try:
            paths, digs = write_sources(src, n, size)
            sizes = [os.path.getsize(p) for p in paths]
            with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=cas) as eng:
                assert eng.import_files(paths, expect=digs) == [(demodel_b200.DM_OK, d) for d in digs]
            shutil.rmtree(src, ignore_errors=True)
            shape = {}
            with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, cas_dir=cas) as eng:
                shape["disk"] = timed_export(eng, base, digs, sizes)
                assert eng.promote(digs) == [demodel_b200.DM_OK] * len(digs)
                shape["hbm"] = timed_export(eng, base, digs, sizes)
                assert shape["hbm"]["d2h_bytes"] == sum(sizes)
            res["shapes"][name] = shape
            print(name, json.dumps(shape), flush=True)
        finally:
            shutil.rmtree(src, ignore_errors=True)
            shutil.rmtree(cas, ignore_errors=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
