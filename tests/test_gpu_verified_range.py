"""dm_cache_open_verified_range on the GPU: the Range: readers of a disk-only blob share one ring load, so N parts of one
blob read and hash the tier file once.  Every byte is checked against hashlib over the same body.

Sizes are module constants so that tests/test_verified_range_host.py can run the same tests over the fake CUDA runtime
with a small arena."""
import hashlib
import os
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 1 << 30             # HBM arena of the engines that have one
RING = 64 << 20             # 64 slabs: a ring-load quarter of 16 slabs, 4 ring loads
SLAB = 1 << 20
BIG = 96 << 20              # larger than SMALL_ARENA
SMALL_ARENA = 16 << 20
IDLE = 16 << 20             # more than a load's 4 slabs: a stalled reader holds its load back
PIECE = 32 << 10            # io.Copy's read size
PARTS = 16
GRACE = 0.5                 # kRangeDetachGrace (engine_cache.cu)


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    kw.setdefault("ring_bytes", RING)
    kw.setdefault("slab_bytes", SLAB)
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


def _read_range(eng, rid, off, end, piece=PIECE):
    """Read [off, end) forward, then the end-of-range read (b"")."""
    got = bytearray()
    while off + len(got) < end:
        part = eng.cache_read(rid, off + len(got), min(piece, end - off - len(got)))
        assert part
        got += part
    assert eng.cache_read(rid, end, piece) == b""
    return bytes(got)


def _clean(eng, max_streams=65536, readers=0):
    for _ in range(1000):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == readers):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _parts(size, n):
    step = -(-size // n)
    return [(k * step, min(step, size - k * step)) for k in range(n) if k * step < size]


def _threads(fns, timeout=300):
    out, errs = [None] * len(fns), []

    def run(i, fn):
        try:
            out[i] = fn()
        except Exception as ex:                                    # reported by the caller
            errs.append(ex)
    th = [threading.Thread(target=run, args=(i, fn)) for i, fn in enumerate(fns)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout)
    assert not any(t.is_alive() for t in th), "a reader did not finish"
    return out, errs


def test_parts_share_one_load(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(1, BIG)
    (dig,) = _populate(cas, [body])
    parts = _parts(BIG, PARTS)
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        total = st0["ring_slabs_total"]
        rids = []
        for off, n in parts:
            rid, size = eng.cache_open_verified_range(dig, off, n)
            assert size == BIG
            rids.append(rid)
        assert eng.stats()["free_stream_slots"] == st0["free_stream_slots"] - 1     # one load's slot
        low = [total]
        stop = threading.Event()

        def sample():
            while not stop.is_set():
                low[0] = min(low[0], eng.stats()["ring_slabs_free"])
                time.sleep(0.002)
        sampler = threading.Thread(target=sample)
        sampler.start()
        got, errs = _threads([lambda rid=rid, off=off, n=n: _read_range(eng, rid, off, off + n)
                              for rid, (off, n) in zip(rids, parts)])
        stop.set()
        sampler.join()
        assert not errs, errs
        assert b"".join(got) == body.tobytes()
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == BIG
        assert st["h2d_bytes"] - st0["h2d_bytes"] == BIG
        assert st["bytes_served"] - st0["bytes_served"] == BIG
        assert low[0] >= total - 4, (low[0], total)
        for rid in rids:
            eng.cache_close(rid)
        _clean(eng)
    with _engine(cas, hbm=SMALL_ARENA) as eng:                      # the same opens as ring loads: refused past the quarter
        share = max(1, eng.stats()["ring_slabs_total"] // 4)
        quarter = share // min(4, share)
        rids, refused = [], 0
        for _ in parts:
            try:
                rids.append(eng.cache_open_verified_ring(dig)[0])
            except demodel_b200.DmError as ex:
                assert ex.code == demodel_b200.DM_ENOMEM
                refused += 1
        assert len(rids) == quarter and refused == len(parts) - quarter
        for rid in rids:
            eng.cache_close(rid)
        _clean(eng)


def test_a_herd_of_whole_blob_readers_is_one_load(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(2, BIG // 2 + 77)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        opened, started = threading.Barrier(4), threading.Barrier(4)

        def reader():
            opened.wait()
            rid, size = eng.cache_open_verified_range(dig)               # four opens at once: one load
            started.wait()
            try:
                return _read_range(eng, rid, 0, size, piece=1 << 20)
            finally:
                eng.cache_close(rid)
        got, errs = _threads([reader] * 4)
        assert not errs, errs
        assert all(g == body.tobytes() for g in got)
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes
        _clean(eng)


def test_a_late_joiner(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(3, BIG)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        first, size = eng.cache_open_verified_range(dig)
        half = size // 2
        got = bytearray()
        while len(got) < half:
            got += eng.cache_read(first, len(got), min(1 << 20, half - len(got)))
        assert bytes(got) == body.tobytes()[:half]
        # the load has given back the slabs below `half`: a reader from 0 starts a load of its own
        late, _ = eng.cache_open_verified_range(dig)
        ahead, _ = eng.cache_open_verified_range(dig, size - (1 << 20))      # ahead of the front: attaches
        got, errs = _threads([lambda: _read_range(eng, first, half, size, piece=1 << 20),
                              lambda: _read_range(eng, late, 0, size, piece=1 << 20),
                              lambda: _read_range(eng, ahead, size - (1 << 20), size)])
        assert not errs, errs
        assert got[0] == body.tobytes()[half:] and got[1] == body.tobytes()
        assert got[2] == body.tobytes()[size - (1 << 20):]
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == 2 * BIG
        for rid in (first, late, ahead):
            eng.cache_close(rid)
        _clean(eng)


def _first_read_then_stall(eng, dig):
    rid, size = eng.cache_open_verified_range(dig)
    first = eng.cache_read(rid, 0, PIECE)
    return rid, size, first


def test_a_stalled_reader_is_detached(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(4, IDLE)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        stalled, size, first = _first_read_then_stall(eng, dig)
        assert first == body.tobytes()[:len(first)]
        other, _ = eng.cache_open_verified_range(dig)
        t0 = time.monotonic()
        assert _read_range(eng, other, 0, size, piece=1 << 20) == body.tobytes()
        assert time.monotonic() - t0 < 120
        pos = len(first)
        assert _read_range(eng, stalled, pos, size, piece=1 << 20) == body.tobytes()[pos:]
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == 2 * IDLE
        for rid in (stalled, other):
            eng.cache_close(rid)
        _clean(eng)


@pytest.mark.parametrize("resume", ["read", "close"])
def test_a_stalled_reader_keeps_pacing_without_budget(tmp_path, resume):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(5, IDLE)
    filler = _body(6, 3 << 20)
    digs = _populate(cas, [body, filler])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        stalled, size, first = _first_read_then_stall(eng, digs[0])
        other, _ = eng.cache_open_verified_range(digs[0])
        hogs = []                                                   # ring loads take the rest of the ring-load quarter
        while True:
            try:
                hogs.append(eng.cache_open_verified_ring(digs[1])[0])
            except demodel_b200.DmError as ex:
                assert ex.code == demodel_b200.DM_ENOMEM
                break
        done = []
        t = threading.Thread(target=lambda: done.append(_read_range(eng, other, 0, size, piece=1 << 20)))
        t.start()
        t.join(GRACE * 4)
        assert t.is_alive() and not done                            # still paced by the stalled reader
        if resume == "read":
            pos = len(first)
            assert _read_range(eng, stalled, pos, size, piece=1 << 20) == body.tobytes()[pos:]
        else:
            eng.cache_close(stalled)
        t.join(120)
        assert not t.is_alive() and done == [body.tobytes()]
        for rid in hogs + [other] + ([stalled] if resume == "read" else []):
            eng.cache_close(rid)
        _clean(eng)


@pytest.mark.parametrize("where", ["middle", "last"])
def test_corrupt_file_fails_every_reader(tmp_path, where):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(7, BIG // 2 + 3)
    (dig,) = _populate(cas, [body])
    path = _blob_file(cas, dig)
    at = body.nbytes // 2 if where == "middle" else body.nbytes - 1
    with open(path, "r+b") as f:
        f.seek(at)
        f.write(bytes([body[at] ^ 0x5A]))
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        parts = _parts(body.nbytes, 4)
        rids = [eng.cache_open_verified_range(dig, off, n)[0] for off, n in parts]

        def reader(rid, off, n):
            """Read the part until its end (b"") or an error: the position reached and the error code."""
            pos = off
            while True:
                try:
                    part = eng.cache_read(rid, pos, PIECE)
                except demodel_b200.DmError as ex:
                    return pos, ex.code
                if not part:
                    return pos, 0
                pos += len(part)
        got, errs = _threads([lambda rid=rid, p=p: reader(rid, *p) for rid, p in zip(rids, parts)])
        assert not errs, errs
        assert all(pos < body.nbytes for pos, _ in got)            # never the last byte
        assert got[-1][1] == demodel_b200.DM_ECORRUPT              # the last part cannot end before the verdict
        for (pos, code), (off, n) in zip(got, parts):
            assert code in (0, demodel_b200.DM_ECORRUPT) and (code or pos == off + n)
        assert not os.path.exists(path) and not os.path.exists(path + ".meta")
        for rid, (pos, _) in zip(rids, got):                       # the verdict reached every reader, and it sticks
            for _ in range(2):
                with pytest.raises(demodel_b200.DmError) as ei:
                    eng.cache_read(rid, pos, PIECE)
                assert ei.value.code == demodel_b200.DM_ECORRUPT
        for rid in rids:
            eng.cache_close(rid)
        assert eng.cache_open_verified_range(dig) is None          # a miss now
        _clean(eng)


def test_close_and_removal(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(8, IDLE)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        rids = [eng.cache_open_verified_range(dig, off, n)[0] for off, n in _parts(IDLE, 4)]
        assert eng.cache_read(rids[0], 0, PIECE) == body.tobytes()[:PIECE]
        assert eng.cache_remove([dig]) == [demodel_b200.DM_ESTATE]
        assert "shared ring load" in eng.error_detail(0)
        for rid in rids[1:]:                                        # all but one: the load keeps running
            eng.cache_close(rid)
        assert eng.stats()["free_stream_slots"] == st0["free_stream_slots"] - 1
        pos, stop = PIECE, _parts(IDLE, 4)[0][1] // 4
        while pos < stop:                                           # part 0 still needs the rest: no verdict yet
            part = eng.cache_read(rids[0], pos, PIECE)
            assert part == body.tobytes()[pos:pos + len(part)] and part
            pos += len(part)
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] < IDLE
        eng.cache_close(rids[0])                                    # the last, before the verdict: the load stops
        _clean(eng)
        assert eng.cache_remove([dig]) == [0]
        assert eng.cache_open_verified_range(dig) is None


@pytest.mark.parametrize("disk_direct", [False, True])
def test_engine_without_hbm_tier(tmp_path, disk_direct):
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    sizes = [0, 1, 63, 64, 4097, 64 << 10, (1 << 20) + 1]
    bodies = [_body(10 + i, n) for i, n in enumerate(sizes)]
    digs = _populate(cas, bodies)
    flags = DM_F_NO_HBM_CAS | (DM_F_DISK_DIRECT if disk_direct else 0)
    with _engine(cas, flags=flags) as eng:
        for body, dig in zip(bodies, digs):
            st0 = eng.stats()
            n = body.nbytes
            ranges = [(0, 0)] + ([(n // 3, n - n // 3 - 1), (n - 1, 1)] if n > 2 else [])
            opened = [(eng.cache_open_verified_range(dig, off, ln), off, ln) for off, ln in ranges]
            got, errs = _threads([lambda o=o, off=off, ln=ln: _read_range(eng, o[0], off, off + (ln or n - off))
                                  for o, off, ln in opened])
            assert not errs, errs
            for g, (o, off, ln) in zip(got, opened):
                assert o[1] == n and g == body.tobytes()[off:off + (ln or n - off)]
            st = eng.stats()
            assert st["bytes_hashed"] - st0["bytes_hashed"] == n     # one load
            assert st["hbm_cas_used"] == 0
            for o, _, _ in opened:
                eng.cache_close(o[0])
        _clean(eng)


def test_blob_in_hbm_opens_as_a_plain_hit(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(20, 3 << 20)
    (dig,) = _populate(cas, [body])
    with _engine(cas) as eng:
        assert eng.promote([dig]) == [0]
        st0 = eng.stats()
        off, n = 1000, 1 << 20
        rid, size = eng.cache_open_verified_range(dig, off, n)
        assert size == body.nbytes
        assert eng.cache_read(rid, off + 5000, 7) == body.tobytes()[off + 5000:off + 5007]     # any order
        assert _read_range(eng, rid, off, off + n) == body.tobytes()[off:off + n]
        assert eng.cache_read(rid, off, 5) == body.tobytes()[off:off + 5]
        for bad in (off - 1, off + n + 1):
            with pytest.raises(demodel_b200.DmError) as ei:
                eng.cache_read(rid, bad, 5)
            assert ei.value.code == demodel_b200.DM_ERANGE
        assert eng.stats()["bytes_hashed"] == st0["bytes_hashed"]
        eng.cache_close(rid)
        _clean(eng)


def test_range_edges(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(30, IDLE)
    (dig,) = _populate(cas, [body])
    size = body.nbytes
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        for off, ln in ((size + 1, 0), (size - 10, 11), (0, size + 1)):
            with pytest.raises(demodel_b200.DmError) as ei:
                eng.cache_open_verified_range(dig, off, ln)
            assert ei.value.code == demodel_b200.DM_ERANGE
        _clean(eng)
        st0 = eng.stats()
        whole, _ = eng.cache_open_verified_range(dig)                    # holds the load back until it reads
        q = size // 4
        mid, _ = eng.cache_open_verified_range(dig, q, q)
        eof, got_size = eng.cache_open_verified_range(dig, size)         # off == size
        assert got_size == size
        for bad in (q - 1, 2 * q + 1):
            with pytest.raises(demodel_b200.DmError) as ei:
                eng.cache_read(mid, bad, 5)
            assert ei.value.code == demodel_b200.DM_ERANGE
        assert eng.cache_read(mid, 2 * q, PIECE) == b""               # the end of a range before the EOF: no wait
        waited = []

        def eof_read():
            waited.append(eng.cache_read(eof, size, PIECE))
            waited.append(eng.stats()["bytes_hashed"] - st0["bytes_hashed"])
        t = threading.Thread(target=eof_read)
        t.start()
        assert _read_range(eng, whole, 0, size, piece=1 << 20) == body.tobytes()
        t.join(120)
        assert waited[0] == b"" and waited[1] >= size                 # the EOF came after the whole blob was hashed
        for rid in (whole, mid, eof):
            eng.cache_close(rid)
        _clean(eng)


def test_ring_and_range_loads_do_not_mix(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(40, 6 << 20)
    (dig,) = _populate(cas, [body])
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        ring, size = eng.cache_open_verified_ring(dig)
        rng, _ = eng.cache_open_verified_range(dig)
        got, errs = _threads([lambda: _read_range(eng, ring, 0, size, piece=1 << 20),
                              lambda: _read_range(eng, rng, 0, size, piece=1 << 20)])
        assert not errs and got == [body.tobytes()] * 2
        assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == 2 * body.nbytes
        eng.cache_close(ring)
        eng.cache_close(rng)
        _clean(eng)


def test_errors_at_open_and_destroy_with_readers_open(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(70, 5 << 20)
    (dig,) = _populate(cas, [body])
    path = _blob_file(cas, dig)
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        assert eng.cache_open_verified_range(hashlib.sha256(b"never cached").digest()) is None
        assert eng._lib.dm_cache_open_verified_range(eng._h, None, 0, 0, None, None) == demodel_b200.DM_EINVAL
        rids = [eng.cache_open_verified_range(dig, off, n)[0] for off, n in _parts(body.nbytes, 3)]
        assert eng.cache_read(rids[0], 0, PIECE) == body.tobytes()[:PIECE]   # one mid-load
    with open(path, "rb") as f:                                        # destroyed with range readers open
        assert hashlib.sha256(f.read()).digest() == dig
