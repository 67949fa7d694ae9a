#!/usr/bin/env python3
"""What following a disk-backed body (dm_cache_follow on a DM_F_DISK_DIRECT stream) costs and saves.

One BODY-byte body over an ARENA-byte arena, so its stream is disk-backed; cas_dir on BASE (tmpfs by default).  The
owner writes it from host memory in 1 MiB pieces, at full speed and throttled to THROTTLE bytes/s, while 0, 1, 8 and 32
followers read it in 32 KiB pieces (io.Copy) from the moment the stream opens.  Reported per setting:
  writer_s        open to the owner's last dm_stream_write returning
  finish_s        open to dm_stream_finish returning (the verdict)
  last_byte_s     per follower: open to its last byte (min / median / max over followers)
  eof_wait_s      per follower: its last byte to its EOF read returning, i.e. waiting for the verdict
  bytes_hashed    dm_stats growth over the run
The same body is then downloaded 1 + N times independently (N = 1 and 8: each its own disk-backed stream, all at once,
at the same speed) for comparison: wall seconds until every dm_stream_finish returned, and bytes_hashed.  Followers are
Python threads; ctypes releases the GIL during each dm_cache_read.  The GPU's name, power limit and SM clocks are read
(nvidia-smi --query-gpu, read-only) in the same run.

usage: disk_follow_probe.py [out.json]     env: BASE (default /dev/shm)
"""
import hashlib
import json
import os
import shutil
import statistics
import sys
import tempfile
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

import demodel_b200  # noqa: E402
from demodel_b200._lib import DM_F_DISK_DIRECT  # noqa: E402
from promote_probe import gpu_info  # noqa: E402

BODY, ARENA, RING = 1 << 30, 256 << 20, 256 << 20
WRITE, READ = 1 << 20, 32 << 10
THROTTLE = 50e6
FOLLOWERS = (0, 1, 8, 32)
INDEPENDENT = (1, 8)


def engine(cas):
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, cas_dir=cas, flags=DM_F_DISK_DIRECT)


def write_body(eng, sid, body, rate, t0):
    for off in range(0, body.nbytes, WRITE):
        if rate:
            lag = t0 + off / rate - time.perf_counter()
            if lag > 0:
                time.sleep(lag)
        eng.stream_write(sid, body[off:off + WRITE])


def followed(base, body, want, rate, n):
    cas = tempfile.mkdtemp(prefix="dm_follow_probe_", dir=base)
    try:
        with engine(cas) as eng:
            h0 = eng.stats()["bytes_hashed"]
            t0 = time.perf_counter()
            sid = eng.stream_open(want, body.nbytes)
            rids = [eng.cache_follow(want)[0] for _ in range(n)]
            last, eof, bad = [0.0] * n, [0.0] * n, []

            def follow(k):
                pos, h = 0, hashlib.sha256()
                while True:
                    piece = eng.cache_read(rids[k], pos, READ)
                    if not piece:
                        eof[k] = time.perf_counter() - t0
                        break
                    h.update(piece)
                    pos += len(piece)
                    last[k] = time.perf_counter() - t0
                if pos != body.nbytes or h.digest() != want:
                    bad.append(k)
                eng.cache_close(rids[k])

            th = [threading.Thread(target=follow, args=(k,)) for k in range(n)]
            for t in th:
                t.start()
            write_body(eng, sid, body, rate, t0)
            writer = time.perf_counter() - t0
            dig, ok = eng.stream_finish(sid)
            finish = time.perf_counter() - t0
            for t in th:
                t.join()
            assert ok and dig == want and not bad, bad
            hashed = eng.stats()["bytes_hashed"] - h0
        r = {"followers": n, "rate_MBps": rate / 1e6 if rate else "full", "writer_s": round(writer, 2),
             "finish_s": round(finish, 2), "bytes_hashed": hashed}
        if n:
            waits = [e - lb for e, lb in zip(eof, last)]
            r["last_byte_s"] = [round(f(last), 2) for f in (min, statistics.median, max)]
            r["eof_wait_s"] = [round(f(waits), 2) for f in (min, statistics.median, max)]
        return r
    finally:
        shutil.rmtree(cas, ignore_errors=True)


def independent(base, body, want, rate, n):
    cas = tempfile.mkdtemp(prefix="dm_follow_probe_ind_", dir=base)
    try:
        with engine(cas) as eng:
            h0 = eng.stats()["bytes_hashed"]
            t0 = time.perf_counter()
            done = []

            def download():
                sid = eng.stream_open(want, body.nbytes)
                write_body(eng, sid, body, rate, t0)
                done.append(eng.stream_finish(sid) == (want, True))

            th = [threading.Thread(target=download) for _ in range(1 + n)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            secs = time.perf_counter() - t0
            assert len(done) == 1 + n and all(done)
            hashed = eng.stats()["bytes_hashed"] - h0
        return {"downloads": 1 + n, "rate_MBps": rate / 1e6 if rate else "full", "wall_s": round(secs, 2),
                "bytes_hashed": hashed}
    finally:
        shutil.rmtree(cas, ignore_errors=True)


def main():
    base = os.environ.get("BASE", "/dev/shm")
    res = {"gpu": gpu_info(), "body": BODY, "arena": ARENA, "base": base, "followed": [], "independent": []}
    body = np.random.default_rng(7).integers(0, 256, BODY, dtype=np.uint8)
    want = hashlib.sha256(body.tobytes()).digest()
    for rate in (0, THROTTLE):
        for n in FOLLOWERS:
            res["followed"].append(followed(base, body, want, rate, n))
            print("followed", res["followed"][-1], flush=True)
        for n in INDEPENDENT:
            if shutil.disk_usage(base).free < (n + 2) * BODY:
                res["independent"].append({"downloads": 1 + n, "skipped": "not enough free space"})
                continue
            res["independent"].append(independent(base, body, want, rate, n))
            print("independent", res["independent"][-1], flush=True)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
