"""Python mirror of the C-ABI, used by tests and bench.py.

Method names follow the hook-side vocabulary of the reference
(demodel/cmd/demodel/start.go:197-204): a response body is *teed*
into a stream (open / write / finish / abort) and a request is answered from
the cache (open / read / close).  All compute happens inside
libdemodel_b200.so; nothing here hashes or copies blob bytes on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Iterable, Iterator, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import (DM_ENOENT, DM_IMP_LINK, DM_ING_FORCE_DEEP, DM_ING_FORCE_WIDE, DM_ING_HASH_ONLY, DM_ING_REPLACE,
                   DM_OK, DM_RM_ALIASES, DM_RM_PARTIAL, DmConfig, DmError, DmStats, check)


def _buf_ptr(buf) -> tuple[C.c_void_p, int]:
    """(pointer, nbytes) of any contiguous bytes-like / numpy array without copying."""
    if isinstance(buf, np.ndarray):
        if not buf.flags["C_CONTIGUOUS"]:
            raise ValueError("array must be C-contiguous")
        return C.c_void_p(buf.ctypes.data), buf.nbytes
    if isinstance(buf, (bytes, bytearray)):
        n = len(buf)
        if isinstance(buf, bytes):
            return C.cast(C.c_char_p(buf), C.c_void_p), n
        return C.cast((C.c_char * n).from_buffer(buf), C.c_void_p), n
    mv = memoryview(buf).cast("B")
    arr = np.frombuffer(mv, dtype=np.uint8)
    return C.c_void_p(arr.ctypes.data), arr.nbytes


def _digest_arg(d: Optional[bytes]):
    if d is None:
        return None
    if len(d) != 32:
        raise ValueError("digest must be 32 bytes")
    return C.cast(C.c_char_p(bytes(d)), C.c_void_p)


class Engine:
    """One engine per GPU (dm_engine_create / dm_engine_destroy)."""

    def __init__(self, device: int = 0, hbm_cas_bytes: int = 1 << 30, ring_bytes: int = 0,
                 slab_bytes: int = 0, max_streams: int = 0, cas_dir: Optional[str] = None, flags: int = 0):
        self._lib = _lib.load()
        cfg = DmConfig()
        cfg.struct_size = C.sizeof(DmConfig)
        cfg.device = device
        cfg.hbm_cas_bytes = hbm_cas_bytes
        cfg.ring_bytes = ring_bytes
        cfg.slab_bytes = slab_bytes
        cfg.max_streams = max_streams
        cfg.cas_dir = cas_dir.encode() if cas_dir else None
        cfg.flags = flags
        handle = C.c_void_p()
        check(self._lib.dm_engine_create(C.byref(cfg), C.byref(handle)), "dm_engine_create")
        self._h = handle
        self.device = device
        self.cas_dir = cas_dir

    # -- lifetime ---------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.dm_engine_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> dict:
        st = DmStats()
        check(self._lib.dm_engine_stats(self._h, C.byref(st)), "dm_engine_stats")
        return {name: getattr(st, name) for name, _ in DmStats._fields_}

    # -- ingest (OnResponse body tee) ---------------------------------------
    def stream_open(self, expect: Optional[bytes] = None, size_hint: int = 0) -> int:
        sid = C.c_uint64()
        check(self._lib.dm_stream_open(self._h, _digest_arg(expect), size_hint, C.byref(sid)), "dm_stream_open")
        return sid.value

    def stream_write(self, sid: int, data) -> None:
        ptr, n = _buf_ptr(data)
        check(self._lib.dm_stream_write(self._h, sid, ptr, n), "dm_stream_write")

    def stream_write_at(self, sid: int, offset: int, data) -> None:
        """One piece of a Range part: bytes for blob offset `offset`, any order."""
        ptr, n = _buf_ptr(data)
        check(self._lib.dm_stream_write_at(self._h, sid, offset, ptr, n), "dm_stream_write_at")

    def stream_checkpoint(self, sid: int) -> tuple[bytes, int]:
        """(32-byte chaining value as 8 native words, bytes hashed) of an open stream."""
        ck = _lib.DmCheckpoint()
        check(self._lib.dm_stream_checkpoint(self._h, sid, C.byref(ck)), "dm_stream_checkpoint")
        return bytes(ck), ck.bytes

    def stream_resume(self, checkpoint: bytes, expect: Optional[bytes] = None, size_hint: int = 0) -> int:
        ck = _lib.DmCheckpoint.from_buffer_copy(checkpoint)
        sid = C.c_uint64()
        check(self._lib.dm_stream_resume(self._h, C.byref(ck), _digest_arg(expect), size_hint, C.byref(sid)),
              "dm_stream_resume")
        return sid.value

    def stream_suspend(self, sid: int) -> int:
        """Save an interrupted download under <cas_dir>/partial and close the stream; returns the byte count
        saved (the proxy re-requests `Range: bytes=<that>-`)."""
        off = C.c_uint64()
        check(self._lib.dm_stream_suspend(self._h, sid, C.byref(off)), "dm_stream_suspend")
        return off.value

    def stream_resume_saved(self, expect: bytes, size_hint: int = 0) -> Optional[tuple[int, int]]:
        """(stream id, resume offset) continuing a download saved by stream_suspend - also after a restart of the
        engine over the same cas_dir - or None when nothing is saved for this digest."""
        sid, off = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_stream_resume_saved(self._h, _digest_arg(expect), size_hint, C.byref(sid), C.byref(off))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_stream_resume_saved")
        return sid.value, off.value

    def error_detail(self, ident: int = 0) -> str:
        """Detail text of the last failing call on stream / reader `ident` (0 = calls without an id)."""
        n = C.c_size_t()
        buf = C.create_string_buffer(1024)
        check(self._lib.dm_error_detail(self._h, ident, buf, 1024, C.byref(n)), "dm_error_detail")
        return buf.value.decode(errors="replace")

    def stream_set_meta(self, sid: int, key: str, value: str) -> None:
        check(self._lib.dm_stream_set_meta(self._h, sid, key.encode(), value.encode()), "dm_stream_set_meta")

    def stream_acquire(self, sid: int) -> tuple[int, int]:
        ptr, cap = C.c_void_p(), C.c_size_t()
        check(self._lib.dm_stream_acquire(self._h, sid, C.byref(ptr), C.byref(cap)), "dm_stream_acquire")
        return ptr.value, cap.value

    def stream_commit(self, sid: int, n: int) -> None:
        check(self._lib.dm_stream_commit(self._h, sid, n), "dm_stream_commit")

    def stream_flush(self, sid: int) -> None:
        check(self._lib.dm_stream_flush(self._h, sid), "dm_stream_flush")

    def stream_finish(self, sid: int) -> tuple[bytes, bool]:
        out = (C.c_uint8 * 32)()
        matched = C.c_int()
        check(self._lib.dm_stream_finish(self._h, sid, out, C.byref(matched)), "dm_stream_finish")
        return bytes(out), bool(matched.value)

    def stream_abort(self, sid: int) -> None:
        check(self._lib.dm_stream_abort(self._h, sid), "dm_stream_abort")

    def ingest(self, data, expect: Optional[bytes] = None, chunk: int = 32768, size_hint: Optional[int] = None
               ) -> tuple[bytes, bool]:
        """Tee one whole body through a stream in `chunk`-byte writes."""
        mv = memoryview(data).cast("B")
        sid = self.stream_open(expect, len(mv) if size_hint is None else size_hint)
        try:
            arr = np.frombuffer(mv, dtype=np.uint8)
            for off in range(0, len(arr), chunk):
                self.stream_write(sid, arr[off:off + chunk])
        except Exception:
            self.stream_abort(sid)
            raise
        try:
            return self.stream_finish(sid)
        except DmError:
            try:
                self.stream_abort(sid)        # some failures leave the stream open; a released id just says so
            except DmError:
                pass
            raise

    # -- hit serving (OnRequest short-circuit) --------------------------------
    def cache_contains(self, digest: bytes) -> Optional[int]:
        size = C.c_uint64()
        rc = self._lib.dm_cache_contains(self._h, _digest_arg(digest), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_contains")
        return size.value

    def cache_open(self, digest: bytes) -> Optional[tuple[int, int]]:
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_cache_open(self._h, _digest_arg(digest), C.byref(rid), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_open")
        return rid.value, size.value

    def cache_open_verified(self, digest: bytes) -> Optional[tuple[int, int]]:
        """dm_cache_open that never serves an unverified disk-tier blob: (reader, size) or None on a miss.

        A blob in HBM opens as with cache_open.  One on the disk tier only is loaded into HBM and hashed there while
        the reader is served from the loaded bytes; the read of the last byte (and the EOF read) waits for the verdict.
        A mismatch makes that read and every later one raise DM_ECORRUPT (file and sidecar are removed); DM_EIO and
        DM_ECUDA likewise.  Raises DM_ENOMEM when the blob cannot be loaded (larger than the arena, no room, no
        slot: cache_open still serves it), DM_ECORRUPT when the file is not its sidecar's size, DM_ESTATE on an
        engine without an HBM tier."""
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_cache_open_verified(self._h, _digest_arg(digest), C.byref(rid), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_open_verified")
        return rid.value, size.value

    def cache_open_verified_ring(self, digest: bytes) -> Optional[tuple[int, int]]:
        """A verified hit that takes no HBM extent: (reader, size) or None on a miss.

        A blob in HBM opens as with cache_open.  One on the disk tier only is read through pinned ring slabs, hashed on
        the GPU as dm_cache_verify hashes it, and the reader is served from those slabs: it works for blobs larger than
        the arena and on engines without an HBM tier.  Reads go forward only (the first may start anywhere; a read
        below the end of the previous one raises DM_ESTATE), and the read of the last byte (and the EOF read) waits
        for the verdict.  A mismatch makes that read and every later one raise DM_ECORRUPT (file and sidecar are
        removed); DM_EIO and DM_ECUDA likewise.  Raises DM_ENOMEM when ring loads hold their share of the ring or no
        stream slot is to spare, DM_ECORRUPT when the file is not its sidecar's size."""
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_cache_open_verified_ring(self._h, _digest_arg(digest), C.byref(rid), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_open_verified_ring")
        return rid.value, size.value

    def cache_open_verified_range(self, digest: bytes, off: int = 0, length: int = 0) -> Optional[tuple[int, int]]:
        """A verified hit on bytes [off, off + length) of a blob (length 0: to the end): (reader, size) or None on a
        miss.  `size` is the whole blob's.

        A blob in HBM opens as with cache_open, its reads kept within the range.  One on the disk tier only is served
        by a shared ring load: the range readers of one blob that a running load can still serve attach to it, so the
        file is read and hashed once for all of them.  Reads stay within the range (DM_ERANGE otherwise) and go forward
        only; the read at off + length returns b"", and when that is the blob's end it waits for the verdict, as the
        read of the last byte does.  A mismatch makes every attached reader's read raise DM_ECORRUPT.  Raises DM_ERANGE
        when the range is not within the blob, DM_ENOMEM when a new load was needed and none can be reserved."""
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_cache_open_verified_range(self._h, _digest_arg(digest), off, length, C.byref(rid),
                                                     C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_open_verified_range")
        return rid.value, size.value

    def cache_follow(self, digest: bytes) -> Optional[tuple[int, int]]:
        """Attach to a body that is still being ingested (request coalescing): (reader, size_hint) or None.

        size_hint is 0 when the body's size is unknown.  Reads block until the bytes have arrived: in HBM, or, for a
        disk-backed body (DM_F_DISK_DIRECT), in its file; the read at EOF waits for the verdict.  A failed, aborted or
        suspended body makes reads raise DM_ESTATE.  None also for a stream that retains nothing to serve."""
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_cache_follow(self._h, _digest_arg(digest), C.byref(rid), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_follow")
        return rid.value, size.value

    def cache_read(self, rid: int, off: int, n: int) -> bytes:
        out = np.empty(n, dtype=np.uint8)
        got = C.c_size_t()
        check(self._lib.dm_cache_read(self._h, rid, off, C.c_void_p(out.ctypes.data), n, C.byref(got)), "dm_cache_read")
        return out[:got.value].tobytes()

    def cache_meta(self, rid: int) -> dict:
        """The blob's sidecar (digest, size, encoding, replayable response headers)."""
        import json
        n = C.c_size_t()
        check(self._lib.dm_cache_meta(self._h, rid, None, 0, C.byref(n)), "dm_cache_meta")
        buf = C.create_string_buffer(n.value + 1)
        check(self._lib.dm_cache_meta(self._h, rid, buf, n.value + 1, C.byref(n)), "dm_cache_meta")
        return json.loads(buf.value.decode())

    def cache_close(self, rid: int) -> None:
        check(self._lib.dm_cache_close(self._h, rid), "dm_cache_close")

    def cache_evict(self, digest: bytes) -> bool:
        rc = self._lib.dm_cache_evict(self._h, _digest_arg(digest))
        if rc == DM_ENOENT:
            return False
        check(rc, "dm_cache_evict")
        return True

    def cache_remove(self, digests: Sequence[bytes], aliases: bool = False, partial: bool = False) -> list[int]:
        """dm_cache_remove: delete blobs from both tiers.  aliases=True also deletes every alias naming a removed
        digest; partial=True also deletes a download of it saved by dm_stream_suspend.  One status per digest: DM_OK,
        DM_ENOENT (on neither tier), DM_ESTATE (being placed or loaded right now, nothing removed: retry later;
        error_detail(0) says what holds it) or DM_EIO."""
        digests = list(digests)
        if any(len(d) != 32 for d in digests):
            raise ValueError("every digest must be 32 bytes")
        status = (C.c_int32 * max(len(digests), 1))()
        blob = b"".join(digests)
        flags = (DM_RM_ALIASES if aliases else 0) | (DM_RM_PARTIAL if partial else 0)
        check(self._lib.dm_cache_remove(self._h, C.cast(C.c_char_p(blob), C.c_void_p) if digests else None,
                                        len(digests), flags, status), "dm_cache_remove")
        return list(status[:len(digests)])

    def promote(self, digests: Sequence[bytes]) -> list[int]:
        """dm_cache_promote: bring cached blobs back into HBM, each disk copy verified on the GPU as it loads.
        One status per digest: DM_OK (in HBM now), DM_ENOENT, DM_ENOMEM, DM_EIO, DM_ECUDA or DM_ECORRUPT (the disk
        copy did not hash to its name and was removed)."""
        digests = list(digests)
        if any(len(d) != 32 for d in digests):
            raise ValueError("every digest must be 32 bytes")
        status = (C.c_int32 * max(len(digests), 1))()
        blob = b"".join(digests)
        check(self._lib.dm_cache_promote(self._h, C.cast(C.c_char_p(blob), C.c_void_p) if digests else None,
                                         len(digests), status), "dm_cache_promote")
        return list(status[:len(digests)])

    def verify(self, digests: Sequence[bytes]) -> list[int]:
        """dm_cache_verify: hash each disk-tier copy in place on the GPU, without loading it into HBM.  One status per
        digest: DM_OK, DM_ENOENT, DM_ECORRUPT (the file did not hash to its name, or did not have its sidecar's
        size, and was removed), DM_EIO, DM_ECUDA or DM_ENOMEM (no stream slot to spare)."""
        digests = list(digests)
        if any(len(d) != 32 for d in digests):
            raise ValueError("every digest must be 32 bytes")
        status = (C.c_int32 * max(len(digests), 1))()
        blob = b"".join(digests)
        check(self._lib.dm_cache_verify(self._h, C.cast(C.c_char_p(blob), C.c_void_p) if digests else None,
                                        len(digests), status), "dm_cache_verify")
        return list(status[:len(digests)])

    def list(self, after: Optional[bytes] = None, cap: int = 4096) -> list[tuple[bytes, int]]:
        """dm_cache_list: up to `cap` (digest, size) pairs of the disk tier in ascending digest order, strictly after
        `after`.  Fewer than `cap` means the listing is complete; page by passing the last digest returned."""
        if cap < 0:
            raise ValueError("cap must be >= 0")
        digs = (C.c_uint8 * (32 * max(cap, 1)))()
        sizes = (C.c_uint64 * max(cap, 1))()
        n = C.c_uint32()
        check(self._lib.dm_cache_list(self._h, _digest_arg(after), digs, sizes, cap, C.byref(n)), "dm_cache_list")
        raw = bytes(digs)
        return [(raw[32 * i:32 * i + 32], sizes[i]) for i in range(n.value)]

    def import_files(self, paths: Sequence[str], expect: Optional[Sequence[Optional[bytes]]] = None,
                     keys: Optional[Sequence[Optional[str]]] = None, link: bool = False) -> list[tuple[int, bytes]]:
        """dm_cache_import: hash files already on the host on the GPU and place them in the disk tier.  expect[i] is
        the SHA-256 paths[i] must hash to, or None when it is not known; keys[i], when not None, is entered in the
        alias index once entry i is cached.  link=True hard-links instead of copying where it can.  One (status,
        digest) per path: DM_OK (digest: its SHA-256), DM_ECORRUPT (digest: what it hashed to), DM_ENOENT, DM_EINVAL
        (not a regular file), DM_EIO, DM_ECUDA or DM_ENOMEM; the digest is 32 zero bytes for the last five."""
        paths = [os.fsencode(p) for p in paths]
        n = len(paths)
        if expect is not None:
            expect = list(expect)
            if len(expect) != n or any(x is not None and len(x) != 32 for x in expect):
                raise ValueError("expect must hold one 32-byte digest or None per path")
        if keys is not None:
            keys = list(keys)
            if len(keys) != n:
                raise ValueError("keys must hold one key or None per path")
        c_paths = (C.c_char_p * max(n, 1))(*paths)
        rows = b"".join(x if x is not None else bytes(32) for x in expect) if expect is not None else None
        c_keys = (C.c_char_p * max(n, 1))(*[k.encode() if k is not None else None for k in keys]) if keys is not None else None
        digs = (C.c_uint8 * (32 * max(n, 1)))()
        status = (C.c_int32 * max(n, 1))()
        check(self._lib.dm_cache_import(self._h, c_paths, C.cast(C.c_char_p(rows), C.c_void_p) if rows else None,
                                        c_keys, n, DM_IMP_LINK if link else 0, digs, status), "dm_cache_import")
        raw = bytes(digs)
        return [(status[i], raw[32 * i:32 * i + 32]) for i in range(n)]

    def export(self, digests: Sequence[bytes], paths: Sequence[str]) -> list[int]:
        """dm_cache_export: write cached blobs to files, each copy hashed on the GPU before it is renamed over
        paths[i] (missing parent directories are created).  The cache is only read.  One status per entry: DM_OK,
        DM_ENOENT (on neither tier), DM_ECORRUPT (the copy did not hash to its name; nothing written, the cache left
        to verify), DM_EIO, DM_ECUDA or DM_ENOMEM.  Raises DM_EINVAL when one path is given two different digests."""
        digests, paths = list(digests), [os.fsencode(p) for p in paths]
        if len(digests) != len(paths) or any(len(d) != 32 for d in digests):
            raise ValueError("one 32-byte digest per path")
        n = len(paths)
        c_paths = (C.c_char_p * max(n, 1))(*paths)
        status = (C.c_int32 * max(n, 1))()
        blob = b"".join(digests)
        check(self._lib.dm_cache_export(self._h, C.cast(C.c_char_p(blob), C.c_void_p) if n else None, c_paths, n,
                                        status), "dm_cache_export")
        return list(status[:n])

    def set_disk_limit(self, limit_bytes: int) -> None:
        """dm_cache_set_disk_limit: keep the disk tier at or under `limit_bytes` (apparent sizes), evicting least
        recently used blobs and saved downloads that nothing pins; 0 turns the limit off.  The first non-zero limit
        walks the tier once to build its index."""
        check(self._lib.dm_cache_set_disk_limit(self._h, limit_bytes), "dm_cache_set_disk_limit")

    def disk_usage(self) -> dict:
        """dm_cache_disk_usage: limit, bytes in use by kind, eviction and refusal counters."""
        u = _lib.DmDiskUsage()
        u.struct_size = C.sizeof(_lib.DmDiskUsage)
        check(self._lib.dm_cache_disk_usage(self._h, C.byref(u)), "dm_cache_disk_usage")
        return {name: getattr(u, name) for name, _ in _lib.DmDiskUsage._fields_ if name not in ("struct_size", "reserved")}

    # -- URL-keyed requests (the OnRequest hook is handed a URL) -----------------------
    def alias_put(self, key: str, digest: bytes) -> None:
        check(self._lib.dm_cache_alias_put(self._h, key.encode(), _digest_arg(digest)), "dm_cache_alias_put")

    def alias_get(self, key: str) -> Optional[bytes]:
        out = (C.c_uint8 * 32)()
        rc = self._lib.dm_cache_alias_get(self._h, key.encode(), out)
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_cache_alias_get")
        return bytes(out)

    def alias_del(self, key: str) -> bool:
        """dm_cache_alias_del: False when the key was not known."""
        rc = self._lib.dm_cache_alias_del(self._h, key.encode())
        if rc == DM_ENOENT:
            return False
        check(rc, "dm_cache_alias_del")
        return True

    def alias_list(self, prefix: str = "", page: int = 1024, keys_bytes: int = 1 << 20) -> Iterator[tuple[str, bytes]]:
        """dm_cache_alias_list, paged: every (key, digest) whose key starts with `prefix`, in ascending byte order of
        the UTF-8 keys.  Each page asks for up to `page` entries in a `keys_bytes` key buffer (a key of up to 4096
        bytes always fits)."""
        if page < 1 or keys_bytes < 4097:
            raise ValueError("page must be >= 1 and keys_bytes >= 4097")
        keys = (C.c_char * keys_bytes)()
        digs = (C.c_uint8 * (32 * page))()
        n, more = C.c_uint32(), C.c_int()
        after = None
        while True:
            check(self._lib.dm_cache_alias_list(self._h, prefix.encode(), after, keys, keys_bytes, digs, page,
                                                C.byref(n), C.byref(more)), "dm_cache_alias_list")
            raw, d, pos = keys.raw, bytes(digs), 0
            for i in range(n.value):
                end = raw.index(b"\0", pos)
                after = raw[pos:end]
                yield after.decode(), d[32 * i:32 * i + 32]
                pos = end + 1
            if not more.value:
                return

    def proxy_fetch(self, url: str, body, expect: Optional[bytes] = None, chunk: int = 32768) -> tuple[bytes, bool]:
        """OnResponse twin for one body fetched under `url` (BodyTee + SetURL): (digest, matched)."""
        ptr, n = _buf_ptr(body)
        out = (C.c_uint8 * 32)()
        matched = C.c_int()
        check(self._lib.dm_proxy_fetch(self._h, url.encode(), ptr, n, _digest_arg(expect), chunk, out, C.byref(matched)),
              "dm_proxy_fetch")
        return bytes(out), bool(matched.value)

    def proxy_request(self, url: str) -> Optional[tuple[int, int]]:
        """OnRequest twin: (reader, size) when the URL names a cached blob (digest in the URL, or alias), else None."""
        rid, size = C.c_uint64(), C.c_uint64()
        rc = self._lib.dm_proxy_request(self._h, url.encode(), C.byref(rid), C.byref(size))
        if rc == DM_ENOENT:
            return None
        check(rc, "dm_proxy_request")
        return rid.value, size.value

    def proxy_manifest(self, body: bytes, content_encoding: Optional[str] = None, chunk: int = 32768, max_layers: int = 64):
        """OnResponse twin for a manifest response: passes the body through, inflates gzip, parses, prefetches.
        Returns [(digest, size, media_type, stream_id)]."""
        layers = (_lib.DmLayer * max_layers)()
        ids = (C.c_uint64 * max_layers)()
        n = C.c_uint32()
        ptr, nbytes = _buf_ptr(body)
        check(self._lib.dm_proxy_manifest(self._h, ptr, nbytes, content_encoding.encode() if content_encoding else None,
                                          chunk, layers, ids, max_layers, C.byref(n)), "dm_proxy_manifest")
        return [(bytes(layers[i].digest), layers[i].size, layers[i].media_type.decode(), ids[i]) for i in range(min(n.value, max_layers))]

    def fetch(self, digest: bytes, chunk: int = 1 << 20) -> Optional[bytes]:
        """Whole cached blob, read the way the hit path would stream it."""
        opened = self.cache_open(digest)
        if opened is None:
            return None
        rid, size = opened
        try:
            parts = [self.cache_read(rid, off, min(chunk, size - off)) for off in range(0, size, chunk)]
        finally:
            self.cache_close(rid)
        return b"".join(parts)

    def cache_device_extents(self, rid: int, max_ext: int = 64) -> list[tuple[int, int]]:
        ptrs = (C.c_void_p * max_ext)()
        lens = (C.c_uint64 * max_ext)()
        n = self._lib.dm_cache_device_extents(self._h, rid, ptrs, lens, max_ext)
        if n < 0:
            check(n, "dm_cache_device_extents")
        return [(ptrs[i], lens[i]) for i in range(min(n, max_ext))]

    # -- device-resident ingest ---------------------------------------------------
    def ingest_device(self, dev_base: int, offsets: Sequence[int], lengths: Sequence[int],
                      expect: Optional[bytes] = None, hash_only: bool = False, replace: bool = False,
                      kernel: Optional[str] = None, raw: bool = False):
        """Hash-and-cache blobs already in HBM: blob i = [dev_base+offsets[i], +lengths[i]).
        Returns (digests, matched, kernel_ms)."""
        off = np.ascontiguousarray(np.asarray(offsets, dtype=np.uint64))
        ln = np.ascontiguousarray(np.asarray(lengths, dtype=np.uint64))
        n = len(off)
        if len(ln) != n:
            raise ValueError("offsets and lengths must have the same length")
        dig = np.zeros(32 * max(n, 1), dtype=np.uint8)
        mat = np.zeros(max(n, 1), dtype=np.uint8)
        ms = C.c_double()
        flags = (DM_ING_HASH_ONLY if hash_only else 0) | (DM_ING_REPLACE if replace else 0)
        if kernel == "wide":
            flags |= DM_ING_FORCE_WIDE
        elif kernel == "deep":
            flags |= DM_ING_FORCE_DEEP
        elif isinstance(kernel, int) and kernel in (1, 2, 4, 8, 16, 32):
            flags |= (kernel.bit_length()) << 8          # DM_ING_SPW: log2(streams per warp) + 1
        elif kernel is not None:
            raise ValueError("kernel must be None, 'wide', 'deep' or streams-per-warp in {1,2,4,8,16,32}")
        exp = None
        if expect is not None:
            if len(expect) != 32 * n:
                raise ValueError("expect must hold n*32 bytes")
            exp = C.cast(C.c_char_p(bytes(expect)), C.c_void_p)
        u64p = C.POINTER(C.c_uint64)
        check(self._lib.dm_ingest_device(self._h, C.c_void_p(dev_base), off.ctypes.data_as(u64p),
                                         ln.ctypes.data_as(u64p), n, exp, C.c_void_p(dig.ctypes.data),
                                         C.c_void_p(mat.ctypes.data), flags, C.byref(ms)), "dm_ingest_device")
        if raw:                               # no per-blob Python objects (large n inside timed loops)
            return dig[:32 * n], mat[:n], ms.value
        digs = [dig[32 * i:32 * i + 32].tobytes() for i in range(n)]
        return digs, [bool(x) for x in mat[:n]], ms.value

    # -- synthetic bytes --------------------------------------------------------------
    def synth_fill_device(self, seed: int, blob: int, byte_off: int, dev_ptr: int, nbytes: int) -> None:
        check(self._lib.dm_synth_fill_device(self._h, seed, blob, byte_off, C.c_void_p(dev_ptr), nbytes),
              "dm_synth_fill_device")

    def synth_fill_device_many(self, seed: int, first_blob: int, dev_base: int, offsets: Sequence[int],
                               lengths: Sequence[int]) -> None:
        off = np.ascontiguousarray(np.asarray(offsets, dtype=np.uint64))
        ln = np.ascontiguousarray(np.asarray(lengths, dtype=np.uint64))
        u64p = C.POINTER(C.c_uint64)
        check(self._lib.dm_synth_fill_device_many(self._h, seed, first_blob, C.c_void_p(dev_base),
                                                  off.ctypes.data_as(u64p), ln.ctypes.data_as(u64p), len(off)),
              "dm_synth_fill_device_many")

    # -- proxy-side driver --------------------------------------------------------------
    def proxy_drive(self, host: np.ndarray, offsets: Sequence[int], expect: Optional[bytes] = None,
                    chunk: int = 32768, concurrency: int = 1, nthreads: int = 0, zero_copy: bool = False
                    ) -> tuple[list[bytes], list[bool], float]:
        off = np.ascontiguousarray(np.asarray(offsets, dtype=np.uint64))
        n = len(off) - 1
        dig = np.zeros(32 * max(n, 1), dtype=np.uint8)
        mat = np.zeros(max(n, 1), dtype=np.uint8)
        secs = C.c_double()
        exp = C.cast(C.c_char_p(bytes(expect)), C.c_void_p) if expect is not None else None
        check(self._lib.dm_proxy_drive(self._h, C.c_void_p(host.ctypes.data), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                       n, exp, chunk, concurrency, nthreads, int(zero_copy),
                                       C.c_void_p(dig.ctypes.data), C.c_void_p(mat.ctypes.data), C.byref(secs)),
              "dm_proxy_drive")
        self.last_drive_verdicts = [int(x) for x in mat[:n]]      # 0 mismatch, 1 matched, 2 aborted by the client
        return [dig[32 * i:32 * i + 32].tobytes() for i in range(n)], [x == 1 for x in mat[:n]], secs.value

    def proxy_serve(self, digests: Iterable[bytes], host_out: np.ndarray, offsets: Sequence[int],
                    chunk: int = 32768, nthreads: int = 1) -> float:
        off = np.ascontiguousarray(np.asarray(offsets, dtype=np.uint64))
        blob = b"".join(digests)
        secs = C.c_double()
        check(self._lib.dm_proxy_serve(self._h, C.cast(C.c_char_p(blob), C.c_void_p), len(off) - 1,
                                       C.c_void_p(host_out.ctypes.data), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                       chunk, nthreads, C.byref(secs)), "dm_proxy_serve")
        return secs.value


def synth_fill_host(seed: int, blob: int, byte_off: int, nbytes: int) -> np.ndarray:
    """Synthetic blob bytes on the host (product generator, not the oracle's)."""
    out = np.empty(nbytes, dtype=np.uint8)
    _lib.load().dm_synth_fill_host(seed, blob, byte_off, C.c_void_p(out.ctypes.data), nbytes)
    return out


def gunzip(data: bytes, cap: int = 1 << 22) -> bytes:
    """dm_gunzip: inflate a gzip / zlib body (manifests served with Content-Encoding: gzip)."""
    out = C.create_string_buffer(max(cap, 1))
    n = C.c_size_t()
    check(_lib.load().dm_gunzip(data, len(data), out, cap, C.byref(n)), "dm_gunzip")
    return out.raw[:n.value]


def shard_of(digest: bytes, n_shards: int) -> int:
    """Which of n_shards engines owns a blob (dm_shard_of)."""
    return int(_lib.load().dm_shard_of(_digest_arg(digest), n_shards))
