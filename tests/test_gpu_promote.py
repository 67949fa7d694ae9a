"""dm_cache_promote on the GPU: blobs that are on the disk tier only (after a restart, or evicted) are loaded back into
HBM and verified by the SHA-256 kernels as they load.  Every body is checked against hashlib over the same bytes; what
the HBM extents hold is copied back with D2H and compared byte for byte.

Sizes are module constants so that tests/test_promote_host.py can run the same tests over the fake CUDA runtime with a
small arena."""
import ctypes as C
import hashlib
import json
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 512 << 20           # HBM arena of the promoting engines
RING = 64 << 20
BIG = 96 << 20              # the one large blob of the round trip
SMALL_ARENA = 16 << 20      # the arena a blob larger than it is promoted on (DM_ENOMEM)
MANY = 3000


def _d2h(ptr, n):
    """Bytes [ptr, ptr + n) of device memory."""
    import torch

    class _Dev:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy().tobytes()


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, ring_bytes=RING, cas_dir=cas, **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _ingest(eng, body, meta=None):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for k, v in (meta or {}).items():
        eng.stream_set_meta(sid, k, v)
    for off in range(0, body.nbytes, 1 << 20):
        eng.stream_write(sid, body[off:off + (1 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _populate(cas, bodies, meta=None):
    """Cache the bodies through ordinary streams, then destroy the engine (its spills drain): all on disk only."""
    with _engine(cas) as eng:
        digs = [_ingest(eng, b, meta) for b in bodies]
    for d, b in zip(digs, bodies):
        assert os.path.getsize(_blob_file(cas, d)) == b.nbytes
    return digs


def _meta_raw(eng, rid):
    n = C.c_size_t()
    assert eng._lib.dm_cache_meta(eng._h, rid, None, 0, C.byref(n)) == 0
    buf = C.create_string_buffer(n.value + 1)
    assert eng._lib.dm_cache_meta(eng._h, rid, buf, n.value + 1, C.byref(n)) == 0
    return buf.raw[:n.value]


def _extents_bytes(eng, rid):
    return b"".join(_d2h(p, n) for p, n in eng.cache_device_extents(rid) if n)


def _read_all(eng, rid, size):
    got = bytearray()
    while len(got) < size:
        part = eng.cache_read(rid, len(got), min(4 << 20, size - len(got)))
        assert part
        got += part
    return bytes(got)


def _on_disk_only(eng, dig):
    import demodel_b200
    rid, _ = eng.cache_open(dig)
    try:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_device_extents(rid)
        assert ei.value.code == demodel_b200.DM_ESTATE
    finally:
        eng.cache_close(rid)


def _check_in_hbm(eng, dig, body):
    rid, size = eng.cache_open(dig)
    try:
        assert size == body.nbytes
        assert _extents_bytes(eng, rid) == body.tobytes()
        assert _read_all(eng, rid, size) == body.tobytes()
    finally:
        eng.cache_close(rid)


def _clean(eng, max_streams=65536, readers=0):
    import time
    for _ in range(400):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == readers):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def test_restart_round_trip(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    sizes = [0, 1, 63, 64, 65, 64 << 10, (64 << 10) + 1, (1 << 20) + 3, BIG]
    bodies = [_body(100 + i, n) for i, n in enumerate(sizes)]
    digs = _populate(cas, bodies, meta={"content-type": "application/octet-stream", "etag": '"v1"'})
    inodes = [os.stat(_blob_file(cas, d)).st_ino for d in digs]
    with _engine(cas) as eng:
        for d in digs:
            _on_disk_only(eng, d)
        st0 = eng.stats()
        assert eng.promote(digs) == [DM_OK] * len(digs)
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == sum(sizes)
        assert st["h2d_bytes"] - st0["h2d_bytes"] >= sum(sizes)
        assert st["hbm_cas_used"] - st0["hbm_cas_used"] >= sum(sizes)
        assert st["blobs_mismatched"] == st0["blobs_mismatched"] and st["d2h_bytes"] == st0["d2h_bytes"]
        assert st["kernel_launches"] > st0["kernel_launches"]
        for d, b in zip(digs, bodies):
            _check_in_hbm(eng, d, b)
            rid, _ = eng.cache_open(d)
            with open(_blob_file(cas, d) + ".meta", "rb") as f:
                assert _meta_raw(eng, rid) == f.read()
            assert eng.cache_meta(rid)["headers"] == {"content-type": "application/octet-stream", "etag": '"v1"'}
            eng.cache_close(rid)
        _clean(eng)
    assert [os.stat(_blob_file(cas, d)).st_ino for d in digs] == inodes        # nothing was spilled again


def test_already_in_hbm_is_not_hashed_again(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body = _body(1, (1 << 20) + 5)
    with _engine(cas) as eng:
        dig = _ingest(eng, body)
        st0 = eng.stats()
        assert eng.promote([dig, dig]) == [DM_OK, DM_OK]
        st = eng.stats()
        assert st["bytes_hashed"] == st0["bytes_hashed"] and st["kernel_launches"] == st0["kernel_launches"]
        assert eng.promote([]) == []


def test_not_cached_no_cas_dir_and_no_hbm_tier(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_ENOENT, DM_ESTATE, DM_OK
    from demodel_b200._lib import DM_F_NO_HBM_CAS
    missing = hashlib.sha256(b"never cached").digest()
    with _engine(str(tmp_path / "cas")) as eng:
        assert eng.promote([missing]) == [DM_ENOENT]
    body = _body(2, 1000)
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING) as eng:     # no cas_dir
        dig = _ingest(eng, body)
        assert eng.promote([missing, dig, missing]) == [DM_ENOENT, DM_OK, DM_ENOENT]
        eng.cache_evict(dig)
        assert eng.promote([dig]) == [DM_ENOENT]
    with _engine(str(tmp_path / "cas2"), flags=DM_F_NO_HBM_CAS) as eng:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.promote([missing])
        assert ei.value.code == DM_ESTATE


def test_corrupt_copies_are_removed_and_a_clean_one_still_promotes(tmp_path):
    from demodel_b200 import DM_ECORRUPT, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(10 + i, (1 << 20) + 3 + i) for i in range(4)]
    flip, trunc, longer, clean = digs = _populate(cas, bodies)
    with open(_blob_file(cas, flip), "r+b") as f:
        f.seek(12345)
        b = f.read(1)
        f.seek(12345)
        f.write(bytes([b[0] ^ 0x01]))
    os.truncate(_blob_file(cas, trunc), bodies[1].nbytes - 100)
    with open(_blob_file(cas, longer), "ab") as f:
        f.write(b"0123456789")
    with _engine(cas) as eng:
        st0 = eng.stats()
        assert eng.promote([flip, trunc, longer, clean]) == [DM_ECORRUPT, DM_ECORRUPT, DM_ECORRUPT, DM_OK]
        # the size mismatches are caught from the sidecar before anything is loaded
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == bodies[0].nbytes + bodies[3].nbytes
        for d in (flip, trunc, longer):
            assert not os.path.exists(_blob_file(cas, d)) and not os.path.exists(_blob_file(cas, d) + ".meta")
            assert eng.cache_contains(d) is None and eng.cache_open(d) is None
        _check_in_hbm(eng, clean, bodies[3])
        # a correct download of the damaged blob caches it again
        assert _ingest(eng, bodies[0]) == flip
        _wait_for_file(cas, flip)
        with open(_blob_file(cas, flip), "rb") as f:
            assert hashlib.sha256(f.read()).digest() == flip
        _clean(eng)
    del digs


def _wait_for_file(cas, dig):
    import time
    for _ in range(500):
        if os.path.exists(_blob_file(cas, dig) + ".meta"):
            return
        time.sleep(0.01)
    raise AssertionError("the blob was not spilled to the disk tier")


def test_blob_without_sidecar_is_promoted_with_no_headers(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body = _body(20, 70000)
    (dig,) = _populate(cas, [body], meta={"etag": '"x"'})
    os.unlink(_blob_file(cas, dig) + ".meta")
    with _engine(cas) as eng:
        assert eng.promote([dig]) == [DM_OK]
        _check_in_hbm(eng, dig, body)
        rid, _ = eng.cache_open(dig)
        meta = eng.cache_meta(rid)
        eng.cache_close(rid)
        assert meta["headers"] == {} and meta["size"] == body.nbytes and meta["digest"] == "sha256:" + dig.hex()


def test_blob_larger_than_the_arena_stays_on_disk(tmp_path):
    from demodel_b200 import DM_ENOMEM
    from demodel_b200._lib import DM_F_DISK_DIRECT
    cas = str(tmp_path / "cas")
    body = _body(21, SMALL_ARENA + 12345)
    with _engine(cas, hbm=SMALL_ARENA, flags=DM_F_DISK_DIRECT) as eng:       # cached on disk by a disk-backed stream
        dig = _ingest(eng, body)
    ino = os.stat(_blob_file(cas, dig)).st_ino
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        assert eng.promote([dig]) == [DM_ENOMEM]
        st = eng.stats()
        assert st["bytes_hashed"] == st0["bytes_hashed"] and st["open_streams"] == 0
        _on_disk_only(eng, dig)
        assert eng.fetch(dig, chunk=4 << 20) == body.tobytes()
    assert os.stat(_blob_file(cas, dig)).st_ino == ino


def test_eviction_after_promotion_serves_from_disk_again(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body = _body(22, (2 << 20) + 7)
    (dig,) = _populate(cas, [body])
    ino = os.stat(_blob_file(cas, dig)).st_ino
    with _engine(cas) as eng:
        assert eng.promote([dig]) == [DM_OK]
        _check_in_hbm(eng, dig, body)
        assert eng.cache_evict(dig)
        _on_disk_only(eng, dig)
        assert eng.fetch(dig) == body.tobytes()
        assert eng.promote([dig]) == [DM_OK]                                # and back again
        _check_in_hbm(eng, dig, body)
        assert eng.cache_evict(dig)
        _clean(eng)
    assert os.stat(_blob_file(cas, dig)).st_ino == ino


def test_many_blobs_share_launches(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    rng = np.random.default_rng(23)
    sizes = rng.integers(1, 8192, MANY)
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    host = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    with _engine(cas) as eng:
        digs, ok, _ = eng.proxy_drive(host, offsets, concurrency=64, nthreads=4)
        assert all(ok)
    with _engine(cas) as eng:
        st0 = eng.stats()
        assert eng.promote(digs) == [DM_OK] * MANY
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == int(offsets[-1])
        assert st["kernel_launches"] - st0["kernel_launches"] < MANY // 10      # the chains went out together
        for i in range(0, MANY, 97):
            _check_in_hbm(eng, digs[i], host[int(offsets[i]):int(offsets[i + 1])])
        _clean(eng)


def test_stream_ingesting_the_same_digest_while_it_is_promoted(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body = _body(24, BIG // 2 + 3)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        out = {}
        t = threading.Thread(target=lambda: out.setdefault("st", eng.promote([dig])))
        t.start()
        assert _ingest(eng, body) == dig
        t.join()
        assert out["st"] == [DM_OK]
        _check_in_hbm(eng, dig, body)
        _clean(eng)
    with open(_blob_file(cas, dig), "rb") as f:
        assert hashlib.sha256(f.read()).digest() == dig


def test_two_threads_promote_overlapping_sets(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(30 + i, (i + 1) * 300001) for i in range(8)]
    digs = _populate(cas, bodies)
    with _engine(cas) as eng:
        res = [None, None]

        def run(k, subset):
            res[k] = eng.promote(subset)
        th = [threading.Thread(target=run, args=(0, digs[:6])), threading.Thread(target=run, args=(1, digs[2:][::-1]))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert res == [[DM_OK] * 6, [DM_OK] * 6]
        for d, b in zip(digs, bodies):
            _check_in_hbm(eng, d, b)
        _clean(eng)


def test_disk_reader_opened_before_promotion_keeps_reading(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body = _body(40, (3 << 20) + 1)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        rid, size = eng.cache_open(dig)
        first = eng.cache_read(rid, 0, 1000)
        assert eng.promote([dig]) == [DM_OK]
        assert first + _read_all(eng, rid, size)[1000:] == body.tobytes()
        eng.cache_close(rid)
        _check_in_hbm(eng, dig, body)
        _clean(eng)


def _damaged_without_sidecar(cas, seed, n):
    """A cached body whose file lost its sidecar and grew 10 bytes (the crash case: nothing but the hash catches it)."""
    body = _body(seed, n)
    (dig,) = _populate(cas, [body])
    os.unlink(_blob_file(cas, dig) + ".meta")
    with open(_blob_file(cas, dig), "ab") as f:
        f.write(b"0123456789")
    return body, dig


def _wait_for_verified_file(cas, dig):
    import time
    for _ in range(500):
        try:
            with open(_blob_file(cas, dig), "rb") as f:
                if hashlib.sha256(f.read()).digest() == dig:
                    return
        except FileNotFoundError:
            pass
        time.sleep(0.01)
    raise AssertionError("the disk tier never got a copy that hashes to its name")


@pytest.mark.parametrize("short_of", ["slots", "arena"])
def test_a_promotion_that_cannot_load_leaves_no_trace(tmp_path, short_of):
    """No slot to spare, or no room in the arena: DM_ENOMEM, and a correct download afterwards is cached with its own
    size (not the damaged file's) and replaces the damaged file."""
    from demodel_b200 import DM_ENOMEM
    cas = str(tmp_path / "cas")
    body, dig = _damaged_without_sidecar(cas, 60, 70000)
    arena = short_of == "arena"
    slots = 8 if arena else 2                               # slots: one held leaves one free, which is not taken
    with _engine(cas, hbm=SMALL_ARENA if arena else None, max_streams=slots) as eng:
        held = eng.stream_open(None, SMALL_ARENA if arena else 0)         # arena: reserves all of it
        assert eng.promote([dig]) == [DM_ENOMEM]
        eng.stream_abort(held)
        assert _ingest(eng, body) == dig
        rid, size = eng.cache_open(dig)
        assert size == body.nbytes and _read_all(eng, rid, size) == body.tobytes()
        eng.cache_close(rid)
        _wait_for_verified_file(cas, dig)
        _clean(eng, max_streams=slots)


def test_stream_and_promotion_of_a_damaged_file_race(tmp_path):
    """A promotion that will find the file bad runs while a stream ingests the correct body.  Whichever publishes
    first, the blob ends up with the stream's size and bytes, and the disk tier with a copy that hashes to its name."""
    from demodel_b200 import DM_ECORRUPT, DM_OK
    cas = str(tmp_path / "cas")
    body, dig = _damaged_without_sidecar(cas, 61, BIG // 2 + 3)
    with _engine(cas) as eng:
        out = {}
        t = threading.Thread(target=lambda: out.setdefault("st", eng.promote([dig])))
        t.start()
        assert _ingest(eng, body) == dig
        t.join()
        assert out["st"] in ([DM_OK], [DM_ECORRUPT])
        _check_in_hbm(eng, dig, body)
        _wait_for_verified_file(cas, dig)
        assert eng.cache_evict(dig)
        assert eng.fetch(dig, chunk=4 << 20) == body.tobytes()                # the disk copy is the right one
        _clean(eng)


def test_the_last_free_stream_slot_stays_with_dm_stream_open(tmp_path):
    from demodel_b200 import DM_ENOMEM, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(62, 1000), _body(63, 2000)]
    digs = _populate(cas, bodies)
    with _engine(cas, max_streams=3) as eng:
        held = [eng.stream_open(None, 0) for _ in range(2)]
        assert eng.promote(digs) == [DM_ENOMEM, DM_ENOMEM]                  # one slot free: it is not taken
        last = eng.stream_open(None, 0)
        for s in held + [last]:
            eng.stream_abort(s)
        held = eng.stream_open(None, 0)                                       # two free: the call may use one
        assert eng.promote(digs) == [DM_OK, DM_OK]
        eng.stream_abort(held)
        for d, b in zip(digs, bodies):
            _check_in_hbm(eng, d, b)
        _clean(eng, max_streams=3)


def test_proxy_streams_open_while_a_large_promotion_runs(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(50, BIG)] + [_body(51 + i, 70000 + i) for i in range(60)]
    digs = _populate(cas, bodies)
    small = _body(49, 5000)
    with _engine(cas, max_streams=8) as eng:
        out = {}
        t = threading.Thread(target=lambda: out.setdefault("st", eng.promote(digs)))
        t.start()
        served = 0
        while t.is_alive() or served == 0:
            sids = [eng.stream_open(None, small.nbytes) for _ in range(4)]        # never DM_ENOMEM
            for s in sids:
                eng.stream_write(s, small)
                assert eng.stream_finish(s)[0] == _sha(small)
            served += 1
        t.join()
        assert out["st"] == [DM_OK] * len(digs)
        _check_in_hbm(eng, digs[0], bodies[0])
        _clean(eng, max_streams=8)
