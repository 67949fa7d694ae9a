"""dm_cache_open_verified_ring on the GPU: a hit on a blob that is on the disk tier only is read through pinned ring slabs,
hashed on the GPU, and served from the same slabs, with no HBM extent: blobs larger than the arena and engines without
an HBM tier get verified hits.  Every body is checked against hashlib over the same bytes.

Sizes are module constants so that tests/test_verified_ring_host.py can run the same tests over the fake CUDA runtime
with a small arena."""
import hashlib
import os
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 1 << 30             # HBM arena of the engines that have one
RING = 64 << 20
BIG = 96 << 20              # larger than SMALL_ARENA
SMALL_ARENA = 16 << 20
IDLE = 16 << 20             # the blob a stalled reader leaves part read on a 4-slab ring
PIECE = 32 << 10            # io.Copy's read size


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    kw.setdefault("ring_bytes", RING)
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, cas_dir=cas, **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for off in range(0, body.nbytes, 4 << 20):
        eng.stream_write(sid, body[off:off + (4 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _populate(cas, bodies):
    """Cache the bodies through ordinary streams, then destroy the engine (its spills drain): all on disk only."""
    with _engine(cas) as eng:
        digs = [_ingest(eng, b) for b in bodies]
    for d, b in zip(digs, bodies):
        assert os.path.getsize(_blob_file(cas, d)) == b.nbytes
    return digs


def _read_all(eng, rid, size, off=0, piece=PIECE):
    got = bytearray()
    while off + len(got) < size:
        part = eng.cache_read(rid, off + len(got), min(piece, size - off - len(got)))
        assert part
        got += part
    assert eng.cache_read(rid, size, piece) == b""           # the EOF read
    return bytes(got)


def _clean(eng, max_streams=65536, readers=0):
    for _ in range(1000):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == readers):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _is_ring_reader(eng, rid):
    import demodel_b200
    try:
        eng.cache_device_extents(rid)
        return False
    except demodel_b200.DmError as ex:
        assert ex.code == demodel_b200.DM_ESTATE
        return True


def test_larger_than_arena(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(1, BIG)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        rid, size = eng.cache_open_verified_ring(dig)
        assert size == BIG and _is_ring_reader(eng, rid)
        assert eng.cache_meta(rid)["size"] == BIG             # the sidecar read at open
        data = bytearray()
        while len(data) < size - 1:
            data += eng.cache_read(rid, len(data), min(PIECE, size - 1 - len(data)))
        last = eng.cache_read(rid, size - 1, PIECE)
        # the last byte came after the verdict: the whole blob had been hashed by then
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == BIG
        assert bytes(data) + last == body.tobytes()
        assert eng.cache_read(rid, size, PIECE) == b""
        st = eng.stats()
        assert st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert st["h2d_bytes"] - st0["h2d_bytes"] >= BIG
        eng.cache_close(rid)
        _clean(eng)
        assert eng.stats()["hbm_cas_used"] == st0["hbm_cas_used"]
    with open(_blob_file(cas, dig), "rb") as f:              # the file stays as it is
        assert hashlib.sha256(f.read()).digest() == dig


@pytest.mark.parametrize("disk_direct", [False, True])
def test_engine_without_hbm_tier(tmp_path, disk_direct):
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    sizes = [0, 1, 63, 64, 4097, 64 << 10, (1 << 20) + 1, BIG // 3 + 5]
    bodies = [_body(10 + i, n) for i, n in enumerate(sizes)]
    digs = _populate(cas, bodies)
    flags = DM_F_NO_HBM_CAS | (DM_F_DISK_DIRECT if disk_direct else 0)
    with _engine(cas, flags=flags) as eng:
        for body, dig in zip(bodies, digs):
            st0 = eng.stats()
            rid, size = eng.cache_open_verified_ring(dig)
            assert size == body.nbytes and _is_ring_reader(eng, rid)
            assert _read_all(eng, rid, size) == body.tobytes()
            st = eng.stats()
            assert st["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes
            assert st["hbm_cas_used"] == 0
            eng.cache_close(rid)
        # a second open is a load of its own: hashed again
        st0 = eng.stats()
        rid, size = eng.cache_open_verified_ring(digs[-1])
        assert _read_all(eng, rid, size, piece=1 << 20) == bodies[-1].tobytes()
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == bodies[-1].nbytes
        eng.cache_close(rid)
        _clean(eng)


def test_blob_in_hbm_opens_as_a_plain_hit(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(20, 3 << 20)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        assert eng.promote([dig]) == [0]
        st0 = eng.stats()
        rid, size = eng.cache_open_verified_ring(dig)
        assert not _is_ring_reader(eng, rid)
        assert _read_all(eng, rid, size) == body.tobytes()
        assert eng.cache_read(rid, 0, 5) == body.tobytes()[:5]   # an HBM reader is not forward only
        assert eng.stats()["bytes_hashed"] == st0["bytes_hashed"]
        eng.cache_close(rid)
        _clean(eng)


@pytest.mark.parametrize("where", ["middle", "last"])
def test_corrupt_file_is_refused_and_removed(tmp_path, where):
    import demodel_b200
    cas = str(tmp_path / "cas")
    bodies = [_body(30, BIG // 2 + 3), _body(31, 1000)]
    digs = _populate(cas, bodies)
    for body, dig in zip(bodies, digs):
        path = _blob_file(cas, dig)
        at = body.nbytes // 2 if where == "middle" else body.nbytes - 1
        with open(path, "r+b") as f:
            f.seek(at)
            f.write(bytes([body[at] ^ 0x5A]))
        with _engine(cas, hbm=SMALL_ARENA) as eng:
            rid, size = eng.cache_open_verified_ring(dig)
            got = bytearray()
            with pytest.raises(demodel_b200.DmError) as ei:
                while True:
                    part = eng.cache_read(rid, len(got), PIECE)
                    assert part, "EOF of a body that does not hash to its name"
                    got += part
            assert ei.value.code == demodel_b200.DM_ECORRUPT
            assert len(got) < size                               # never the last byte
            with pytest.raises(demodel_b200.DmError) as ei:      # sticky
                eng.cache_read(rid, len(got), PIECE)
            assert ei.value.code == demodel_b200.DM_ECORRUPT
            assert not os.path.exists(path) and not os.path.exists(path + ".meta")
            eng.cache_close(rid)
            assert eng.cache_open_verified_ring(dig) is None     # a miss now
            _clean(eng)


def test_forward_only_and_range_first_read(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(40, BIG)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        rid, size = eng.cache_open_verified_ring(dig)
        start = size // 2 + 12345                               # Range: bytes=start-
        first = eng.cache_read(rid, start, PIECE)
        assert first == body.tobytes()[start:start + len(first)] and first
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_read(rid, start, PIECE)                   # below the end of the previous read
        assert ei.value.code == demodel_b200.DM_ESTATE
        assert "forward" in eng.error_detail(rid)
        pos = start + len(first)
        assert _read_all(eng, rid, size, off=pos, piece=1 << 20) == body.tobytes()[pos:]
        eng.cache_close(rid)
        _clean(eng)


def test_stalled_reader_does_not_stop_other_streams(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(50, IDLE)
    (dig,) = _populate(cas, [body])
    with demodel_b200.Engine(device=0, hbm_cas_bytes=SMALL_ARENA, ring_bytes=4 << 20, slab_bytes=1 << 20, cas_dir=cas) as eng:
        rid, size = eng.cache_open_verified_ring(dig)
        assert eng.cache_read(rid, 0, PIECE) == body.tobytes()[:PIECE]
        done = []

        def other():
            for k in range(3):
                live = _body(51 + k, (3 << 20) + 17 * k)
                done.append(_ingest(eng, live) == _sha(live))
        t = threading.Thread(target=other)
        t.start()
        t.join(120)                                             # the reader stalls meanwhile
        assert not t.is_alive() and done == [True, True, True]
        assert _read_all(eng, rid, size, off=PIECE, piece=1 << 20) == body.tobytes()[PIECE:]
        eng.cache_close(rid)
        _clean(eng)


def test_ring_share_and_close_before_the_verdict(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(60, IDLE)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        total = eng.stats()["ring_slabs_total"]
        share = max(1, total // 4)
        loads = share // min(4, share)
        rids = []
        for _ in range(loads):
            rid, _size = eng.cache_open_verified_ring(dig)
            rids.append(rid)
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_open_verified_ring(dig)
        assert ei.value.code == demodel_b200.DM_ENOMEM
        assert eng.stats()["ring_slabs_free"] >= total - share    # stalled loads hold their share, no more
        # a running load keeps dm_cache_remove off the digest
        assert eng.cache_remove([dig]) == [demodel_b200.DM_ESTATE]
        assert "ring load" in eng.error_detail(0)
        assert eng.cache_read(rids[0], 0, PIECE) == body.tobytes()[:PIECE]
        for rid in rids:                                        # before their verdicts
            eng.cache_close(rid)
        _clean(eng)
        rid, size = eng.cache_open_verified_ring(dig)           # the share is back
        assert _read_all(eng, rid, size, piece=1 << 20) == body.tobytes()
        eng.cache_close(rid)
        _clean(eng)
        assert eng.cache_remove([dig]) == [0]
        assert eng.cache_open_verified_ring(dig) is None


def test_errors_at_open_and_destroy_with_readers_open(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(70, 5 << 20)
    (dig,) = _populate(cas, [body])
    path = _blob_file(cas, dig)
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        assert eng.cache_open_verified_ring(hashlib.sha256(b"never cached").digest()) is None
        assert eng._lib.dm_cache_open_verified_ring(eng._h, None, None, None) == demodel_b200.DM_EINVAL
        with open(path, "ab") as f:                             # not the size its sidecar states
            f.write(b"x")
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_open_verified_ring(dig)
        assert ei.value.code == demodel_b200.DM_ECORRUPT
        assert not os.path.exists(path)
        _clean(eng)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:                  # destroyed with ring readers open, one mid-load
        rid, size = eng.cache_open_verified_ring(dig)
        assert eng.cache_read(rid, 0, PIECE) == body.tobytes()[:PIECE]
        assert eng.cache_open(dig) is not None
    with open(path, "rb") as f:
        assert hashlib.sha256(f.read()).digest() == dig
