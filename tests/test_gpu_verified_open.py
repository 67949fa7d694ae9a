"""dm_cache_open_verified on the GPU: a hit on a blob that is on the disk tier only is loaded into HBM and hashed there
while the reader is served from the loaded bytes, and no read hands out the last byte before the verdict.  Every body is
checked against hashlib over the same bytes; what the HBM extents hold afterwards is copied back with D2H and compared.

Sizes are module constants so that tests/test_verified_open_host.py can run the same tests over the fake CUDA runtime
with a small arena."""
import ctypes as C
import hashlib
import os
import random
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 1 << 30             # HBM arena of the serving engines
RING = 64 << 20
BIG = 96 << 20              # the large blob of the parity test, and of the corruption and arena-limit tests
GATE = 256 << 20            # the blob whose last byte is checked against its publication
COAL = 64 << 20             # the blob 8 readers open at once
SMALL_ARENA = 16 << 20      # an arena BIG does not fit
IDLE = 16 << 20             # the blob an idle reader leaves half read on a 4-slab ring
PIECE = 32 << 10            # io.Copy's read size


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


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    eng.stream_set_meta(sid, "content-type", "application/octet-stream")
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


def _meta_raw(eng, rid):
    n = C.c_size_t()
    assert eng._lib.dm_cache_meta(eng._h, rid, None, 0, C.byref(n)) == 0
    buf = C.create_string_buffer(n.value + 1)
    assert eng._lib.dm_cache_meta(eng._h, rid, buf, n.value + 1, C.byref(n)) == 0
    return buf.raw[:n.value]


def _extents_bytes(eng, rid):
    return b"".join(_d2h(p, n) for p, n in eng.cache_device_extents(rid) if n)


def _read_all(eng, rid, size, piece=PIECE):
    got = bytearray()
    while len(got) < size:
        part = eng.cache_read(rid, len(got), min(piece, size - len(got)))
        assert part
        got += part
    assert eng.cache_read(rid, size, piece) == b""           # the EOF read
    return bytes(got)


def _in_hbm(eng, dig):
    import demodel_b200
    opened = eng.cache_open(dig)
    if opened is None:
        return False
    try:
        eng.cache_device_extents(opened[0])
        return True
    except demodel_b200.DmError:
        return False
    finally:
        eng.cache_close(opened[0])


def _clean(eng, max_streams=65536, readers=0):
    for _ in range(1000):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == readers):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def test_parity_across_sizes(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    sizes = [0, 1, 63, 64, 65, 64 << 10, (64 << 10) + 1, (1 << 20) - 1, (1 << 20) + 1, BIG]
    bodies = [_body(10 + i, n) for i, n in enumerate(sizes)]
    digs = _populate(cas, bodies)
    rng = random.Random(5)
    with _engine(cas) as eng:
        st0 = eng.stats()
        for d, b in zip(digs, bodies):
            rid, size = eng.cache_open_verified(d)
            assert size == b.nbytes
            with open(_blob_file(cas, d) + ".meta", "rb") as f:
                side = f.read()
            assert _meta_raw(eng, rid) == side                # before the verdict: the sidecar read at open
            if size > 1:
                with pytest.raises(demodel_b200.DmError) as ei:
                    eng.cache_device_extents(rid)
                assert ei.value.code == demodel_b200.DM_ESTATE
                for _ in range(4):                            # random pieces that end before the last byte
                    off = rng.randrange(size - 1)
                    n = rng.randrange(1, size - off)
                    part = eng.cache_read(rid, off, n)
                    assert part and part == b.tobytes()[off:off + len(part)]
            assert hashlib.sha256(_read_all(eng, rid, size)).digest() == d
            assert _extents_bytes(eng, rid) == b.tobytes()
            assert _meta_raw(eng, rid) == side                # after it: the sidecar's text, unchanged
            eng.cache_close(rid)
            assert _in_hbm(eng, d)
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == sum(sizes)
        assert st["blobs_mismatched"] == st0["blobs_mismatched"]
        _clean(eng)


def test_last_byte_only_after_publication(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(20, GATE)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        rid, size = eng.cache_open_verified(dig)
        off, piece = 0, 4 << 20
        while off < size - 1:
            part = eng.cache_read(rid, off, min(piece, size - 1 - off))
            assert part == body.tobytes()[off:off + len(part)]
            off += len(part)
        last = eng.cache_read(rid, size - 1, 1)
        probe = eng.cache_open(dig)                            # right after the last byte: the blob is published
        try:
            assert eng.cache_device_extents(probe[0])
        finally:
            eng.cache_close(probe[0])
        assert last == body.tobytes()[-1:]
        assert eng.cache_read(rid, size, 1) == b""
        eng.cache_close(rid)
        _clean(eng)


@pytest.mark.parametrize("case", ["big-middle", "big-last", "tiny-middle", "tiny-last"])
def test_corrupt_tier_file(tmp_path, case):
    import demodel_b200
    cas = str(tmp_path / "cas")
    n = BIG if case.startswith("big") else 1000
    body = _body(30, n)
    other = _body(31, 5000)
    dig, odig = _populate(cas, [body, other])
    path = _blob_file(cas, dig)
    bad = bytearray(body.tobytes())
    bad[n // 2 if case.endswith("middle") else n - 1] ^= 0x5A
    with open(path, "r+b") as f:                               # same size, one byte flipped
        f.seek(n // 2 if case.endswith("middle") else n - 1)
        f.write(bytes([bad[n // 2 if case.endswith("middle") else n - 1]]))
    # the extra file whose size is not its sidecar's
    with open(_blob_file(cas, odig), "ab") as f:
        f.write(b"x")
    with _engine(cas) as eng:
        rid, size = eng.cache_open(dig)                        # the control: a plain open serves the damaged file whole
        assert _read_all(eng, rid, size, 4 << 20) == bytes(bad)
        eng.cache_close(rid)
        rid, size = eng.cache_open_verified(dig)
        assert size == n
        if case.startswith("big"):
            got = bytearray()
            while len(got) < n - 1:                            # everything before the last byte is served
                part = eng.cache_read(rid, len(got), min(4 << 20, n - 1 - len(got)))
                assert part
                got += part
            assert bytes(got) == bytes(bad[:n - 1])
        else:                                                  # a tiny blob lands in HBM with its verdict (a pack)
            with pytest.raises(demodel_b200.DmError) as ei:
                eng.cache_read(rid, 0, n - 1)
            assert ei.value.code == demodel_b200.DM_ECORRUPT
        for off in (n - 1, 0, n):                              # the last byte, and every read after it, fail
            with pytest.raises(demodel_b200.DmError) as ei:
                eng.cache_read(rid, off, 1)
            assert ei.value.code == demodel_b200.DM_ECORRUPT
        assert "hash" in eng.error_detail(rid)
        eng.cache_close(rid)
        assert not os.path.exists(path) and not os.path.exists(path + ".meta")
        assert eng.cache_contains(dig) is None
        assert eng.cache_open_verified(dig) is None
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_open_verified(odig)
        assert ei.value.code == demodel_b200.DM_ECORRUPT
        assert not os.path.exists(_blob_file(cas, odig))
        _clean(eng)


def test_concurrent_opens_share_one_load(tmp_path):
    cas = str(tmp_path / "cas")
    body, body2 = _body(40, COAL), _body(41, COAL)
    dig, dig2 = _populate(cas, [body, body2])
    with _engine(cas) as eng:
        st0 = eng.stats()
        start = threading.Barrier(8)
        results, errors = [None] * 8, []

        def reader(k):
            try:
                start.wait()
                rid, size = eng.cache_open_verified(dig)
                results[k] = _read_all(eng, rid, size, 1 << 20)
                eng.cache_close(rid)
            except Exception as ex:                            # surfaced below
                errors.append(ex)
        th = [threading.Thread(target=reader, args=(k,)) for k in range(8)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        assert all(r == body.tobytes() for r in results)
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == COAL
        assert st["h2d_bytes"] - st0["h2d_bytes"] == COAL
        # a promotion and a follow of a digest under a load
        rid, size = eng.cache_open_verified(dig2)
        assert eng.cache_follow(dig2) is None
        assert eng.promote([dig2]) == [0]
        assert _read_all(eng, rid, size, 1 << 20) == body2.tobytes()
        eng.cache_close(rid)
        st2 = eng.stats()
        assert st2["bytes_hashed"] - st["bytes_hashed"] == COAL
        _clean(eng)


def test_errors_at_open(tmp_path):
    import demodel_b200
    from demodel_b200._lib import DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    body = _body(50, BIG)
    (dig,) = _populate(cas, [body])
    path = _blob_file(cas, dig)
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_open_verified(dig)
        assert ei.value.code == demodel_b200.DM_ENOMEM
        opened = eng.cache_open(dig)                           # the fall-back still serves it
        assert opened and opened[1] == BIG
        eng.cache_close(opened[0])
        assert eng.cache_open_verified(hashlib.sha256(b"never cached").digest()) is None
        _clean(eng)
    with open(path, "rb") as f:
        assert hashlib.sha256(f.read()).digest() == dig
    incoming = os.path.join(cas, "incoming")
    assert not os.path.isdir(incoming) or not os.listdir(incoming)
    with _engine(str(tmp_path / "cas2"), flags=DM_F_NO_HBM_CAS) as eng:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_open_verified(dig)
        assert ei.value.code == demodel_b200.DM_ESTATE


def test_idle_reader_holds_no_ring_and_close_keeps_the_load(tmp_path):
    cas = str(tmp_path / "cas")
    body, live = _body(60, IDLE), _body(61, 4 * IDLE // 3 + 7)
    (dig,) = _populate(cas, [body])
    import demodel_b200
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=4 << 20, slab_bytes=1 << 20, cas_dir=cas) as eng:
        rid, size = eng.cache_open_verified(dig)
        assert eng.cache_read(rid, 0, PIECE) == body.tobytes()[:PIECE]
        _ingest(eng, live)                                     # another body goes through the ring meanwhile
        assert _in_hbm(eng, _sha(live))
        eng.cache_close(rid)                                   # mid-load: the load goes on
        for _ in range(3000):
            if _in_hbm(eng, dig):
                break
            time.sleep(0.01)
        assert _in_hbm(eng, dig)
        rid, size = eng.cache_open(dig)
        assert _extents_bytes(eng, rid) == body.tobytes()
        eng.cache_close(rid)
        _clean(eng)


def test_disk_limit_does_not_evict_a_loading_blob(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(70, COAL)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        rid, size = eng.cache_open_verified(dig)
        eng.set_disk_limit(1)
        assert _read_all(eng, rid, size, 1 << 20) == body.tobytes()
        eng.cache_close(rid)
        assert os.path.exists(_blob_file(cas, dig))
        assert _in_hbm(eng, dig)
        _clean(eng)


def test_restart_verifies_again(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(80, COAL + 12345)
    (dig,) = _populate(cas, [body])
    for _ in range(2):
        with _engine(cas) as eng:
            st0 = eng.stats()
            rid, size = eng.cache_open_verified(dig)
            assert _read_all(eng, rid, size, 1 << 20) == body.tobytes()
            assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes
            eng.cache_close(rid)
            _clean(eng)
    with _engine(cas) as eng:                                  # destroyed with a load running and its reader open
        rid, size = eng.cache_open_verified(dig)
        assert eng.cache_read(rid, 0, PIECE) == body.tobytes()[:PIECE]
    with open(_blob_file(cas, dig), "rb") as f:
        assert hashlib.sha256(f.read()).digest() == dig
