#!/usr/bin/env python3
"""sha256sum-compatible digest of files, computed by the GPU engine (one stream per file, all
files in flight together so the multi-buffer kernel has something to batch).

    python tools/dm_sha256sum.py [--device 0] [--check SUMS] FILE...

Needs a CUDA device: there is no CPU fallback on the hash path.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import demodel_b200  # noqa: E402


def digest_files(eng, paths, chunk=1 << 20):
    opened = []
    for p in paths:
        f = open(p, "rb")
        size = os.fstat(f.fileno()).st_size
        opened.append((p, f, eng.stream_open(None, size)))
    live = list(opened)
    buf = bytearray(chunk)
    while live:                                   # round-robin one piece per file per turn
        nxt = []
        for p, f, sid in live:
            n = f.readinto(buf)
            if n:
                eng.stream_write(sid, memoryview(buf)[:n])
                nxt.append((p, f, sid))
            else:
                eng.stream_flush(sid)
                f.close()
        live = nxt
    return [(p, eng.stream_finish(sid)[0].hex()) for p, _, sid in opened]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--check", help="verify against a sha256sum-format file instead of printing")
    ap.add_argument("files", nargs="*")
    args = ap.parse_args()
    want = {}
    files = list(args.files)
    if args.check:
        for ln in open(args.check):
            d, _, name = ln.strip().partition("  ")
            if name:
                want[name] = d
        files = files or list(want)
    total = sum(os.path.getsize(p) for p in files)
    with demodel_b200.Engine(device=args.device, hbm_cas_bytes=total + (256 << 20), ring_bytes=256 << 20,
                             max_streams=max(4096, len(files) + 16)) as eng:
        bad = 0
        for p, d in digest_files(eng, files):
            if args.check:
                ok = want.get(p) == d
                bad += not ok
                print(f"{p}: {'OK' if ok else 'FAILED'}")
            else:
                print(f"{d}  {p}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
