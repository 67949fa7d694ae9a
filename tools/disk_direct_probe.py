#!/usr/bin/env python3
"""What a client sees when it sends bodies larger than the HBM arena, with and without DM_F_DISK_DIRECT.

Bodies of SIZE bytes (default 192 MiB, arena 64 MiB) are fed from host memory in 32 KiB writes, 1, 4 and 16 at
once (one thread per body), with cas_dir on /dev/shm and on the local temporary directory.  Without the flag
such a body is verify-only: its slabs return to the ring only after their hash job, so the client is held to the
per-stream hash rate.  With it the slabs return once written to the file.  Per case:
  writer_s       wall time of the writes (open .. last write returns): what the client waits for
  writer_GBps    bytes / writer_s
  lag_s          last write returned .. dm_stream_finish returned (hash of the tail + publication)
  hashed_GBps    bytes / (open .. last finish)
The GPU's name, power limit and SM clocks are read (nvidia-smi --query-gpu, read-only) in the same run.

usage: disk_direct_probe.py [out.json]       env: SIZE (bytes per body), RING (ring bytes, default 32 MiB),
                                             LOCAL (directory for the local-disk case)
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
from demodel_b200._lib import DM_F_DISK_DIRECT  # noqa: E402

ARENA = 64 << 20
RING = int(os.environ.get("RING", 32 << 20))     # well below a body: a ring that holds the whole body hides the back-pressure
SIZE = int(os.environ.get("SIZE", 192 << 20))
CHUNK = 32 << 10


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as ex:                         # reported, not fatal: the numbers then lack their context
        return {"error": str(ex)}


def one_case(root, flags, n, body):
    shutil.rmtree(root, ignore_errors=True)
    eng = demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, cas_dir=root, flags=flags)
    done_write, done_finish, errors = [0.0] * n, [0.0] * n, []
    barrier = threading.Barrier(n + 1)

    def client(i):
        try:
            barrier.wait()
            sid = eng.stream_open(None, body.nbytes)
            for off in range(0, body.nbytes, CHUNK):
                eng.stream_write(sid, body[off:off + CHUNK])
            done_write[i] = time.perf_counter()
            eng.stream_flush(sid)
            _, ok = eng.stream_finish(sid)
            done_finish[i] = time.perf_counter()
            assert ok
        except Exception as ex:
            errors.append(ex)
    th = [threading.Thread(target=client, args=(i,)) for i in range(n)]
    for t in th:
        t.start()
    barrier.wait()
    t0 = time.perf_counter()
    for t in th:
        t.join()
    st = eng.stats()
    eng.close()
    shutil.rmtree(root, ignore_errors=True)
    if errors:
        raise errors[0]
    writer_s = max(done_write) - t0
    total = n * body.nbytes
    return {"streams": n, "bytes": total, "writer_s": round(writer_s, 3), "writer_GBps": round(total / writer_s / 1e9, 3),
            "lag_s": round(max(f - w for f, w in zip(done_finish, done_write)), 3),
            "hashed_GBps": round(total / (max(done_finish) - t0) / 1e9, 3), "ring_waits": st["ring_waits"]}


def main():
    body = np.random.default_rng(1).integers(0, 256, SIZE, dtype=np.uint8)
    places = {"/dev/shm": "/dev/shm", "local": os.environ.get("LOCAL", tempfile.gettempdir())}
    res = {"gpu": gpu_info(), "arena_bytes": ARENA, "ring_bytes": RING, "body_bytes": SIZE, "write_bytes": CHUNK, "cases": []}
    for where, base in places.items():
        for n in (1, 4, 16):
            if not os.path.isdir(base) or shutil.disk_usage(base).free < 2 * n * SIZE:
                res["cases"].append({"where": where, "streams": n, "skipped": "not enough free space"})
                continue
            for flag in (0, DM_F_DISK_DIRECT):
                root = tempfile.mkdtemp(prefix="dm_disk_probe_", dir=base)
                r = one_case(root, flag, n, body)
                r.update(where=where, disk_direct=bool(flag))
                res["cases"].append(r)
                print(json.dumps(r), flush=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
