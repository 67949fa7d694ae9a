"""The disk tier under a size limit (dm_cache_set_disk_limit, dm_cache_disk_usage): least recently used blobs and saved
downloads are evicted at every placement, pinned ones never.  Every body is checked against hashlib, and after each
test every file left under blobs/ is hashed on the GPU by dm_cache_verify and must be DM_OK, and used_bytes must equal
a walk of blobs/, incoming/ and partial/.

Sizes are module constants so that tests/test_disk_limit_host.py can run the same tests over the fake CUDA runtime with
a small ring and arena."""
import ctypes as C
import hashlib
import os
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 256 << 20           # HBM arena of the engines
RING = 64 << 20
SLAB = 1 << 20
BLOB = 1 << 20              # one cached body
N = 8                       # bodies per population
SMALL_ARENA = 2 << 20       # the arena a disk-backed body is larger than


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    kw.setdefault("ring_bytes", RING)
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, slab_bytes=SLAB, cas_dir=cas, **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _entry_bytes(cas, dig):
    p = _blob_file(cas, dig)
    return os.path.getsize(p) + (os.path.getsize(p + ".meta") if os.path.exists(p + ".meta") else 0)


def _walk(cas):
    total = 0
    for sub in ("blobs", "incoming", "partial"):
        for root, _, files in os.walk(os.path.join(cas, sub)):
            for f in files:
                p = os.path.join(root, f)
                if os.path.isfile(p) and not os.path.islink(p):
                    total += os.path.getsize(p)
    return total


def _incoming(cas):
    d = os.path.join(cas, "incoming")
    return os.listdir(d) if os.path.isdir(d) else []


def _ingest(eng, body, expect=True, size_hint=True, chunk=1 << 20):
    sid = eng.stream_open(_sha(body) if expect else None, body.nbytes if size_hint else 0)
    for off in range(0, body.nbytes, chunk):
        eng.stream_write(sid, body[off:off + chunk])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _read_all(eng, dig):
    got = eng.cache_open(dig)
    assert got is not None
    rid, size = got
    try:
        out = bytearray()
        while len(out) < size:
            part = eng.cache_read(rid, len(out), min(4 << 20, size - len(out)))
            assert part
            out += part
        return bytes(out)
    finally:
        eng.cache_close(rid)


def _clean(eng, max_streams=65536):
    for _ in range(500):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == 0):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _check_tier(eng, cas):
    """Quiescent: every blob file hashes to its name on the GPU, and the index agrees with the directory walk."""
    import demodel_b200
    _clean(eng)
    u = eng.disk_usage()
    for _ in range(500):                                           # spills run after dm_stream_finish returns
        if not u["limit_bytes"] or u["used_bytes"] == _walk(cas):
            break
        time.sleep(0.01)
        u = eng.disk_usage()
    digs = [d for d, _ in eng.list(cap=1 << 16)]
    assert eng.verify(digs) == [demodel_b200.DM_OK] * len(digs)
    if u["limit_bytes"]:
        assert u["used_bytes"] == _walk(cas), (u, _walk(cas))
        assert u["used_bytes"] == u["blob_bytes"] + u["staging_bytes"] + u["partial_bytes"]
        assert u["blob_files"] == len(digs)
    _clean(eng)


def _disk_only(eng, bodies):
    """Cache the bodies (spilled before finish returns) and take them out of HBM in order: disk-only, ranked 0..n-1."""
    digs = [_ingest(eng, b) for b in bodies]
    for d in digs:
        assert eng.cache_evict(d)
    return digs


def _present(cas, digs):
    return [os.path.exists(_blob_file(cas, d)) for d in digs]


def _evict_one_at_a_time(eng, cas, expect_order):
    """Lower the limit one entry at a time: exactly the next digest of `expect_order` goes each time."""
    for k, d in enumerate(expect_order):
        eng.set_disk_limit(eng.disk_usage()["used_bytes"] - 1)
        assert not os.path.exists(_blob_file(cas, d)), f"step {k}: {d.hex()[:12]} should have gone"
        for later in expect_order[k + 1:]:
            assert os.path.exists(_blob_file(cas, later)), f"step {k}: {later.hex()[:12]} went too early"


def test_lru_order_aliases_and_misses(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(100 + i, BLOB + 64 * i) for i in range(N)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(1 << 50)
        digs = _disk_only(eng, bodies)
        for i, d in enumerate(digs):
            eng.alias_put(f"https://example.test/blob/{i}", d)
        touched = [1, 4, 6]
        for i in touched:
            assert _read_all(eng, digs[i]) == bodies[i].tobytes()
        assert eng.verify(digs) == [demodel_b200.DM_OK] * N       # not a use
        eng.cache_contains(digs[0])                                # not a use
        eng.list()                                                 # not a use
        order = [digs[i] for i in range(N) if i not in touched] + [digs[i] for i in touched]
        used = eng.disk_usage()["used_bytes"]
        assert used == _walk(cas)
        eng.set_disk_limit(used // 2)                              # about half
        u = eng.disk_usage()
        assert u["used_bytes"] <= used // 2 and u["evicted_files"] > 0
        gone = order[:u["evicted_files"]]
        kept = order[u["evicted_files"]:]
        assert not any(_present(cas, gone)) and all(_present(cas, kept))
        for d in gone:
            assert eng.cache_contains(d) is None
            assert eng.cache_open(d) is None
            i = digs.index(d)
            assert eng.alias_get(f"https://example.test/blob/{i}") == d
        for d in kept:
            assert _read_all(eng, d) == bodies[digs.index(d)].tobytes()
        _check_tier(eng, cas)


def test_order_survives_restart_and_verify(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(200 + i, BLOB) for i in range(N)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(1 << 50)
        digs = _disk_only(eng, bodies)
        for i in (5, 0, 3):                                        # these three become the most recent, in this order
            assert _read_all(eng, digs[i]) == bodies[i].tobytes()
    order = [digs[i] for i in (1, 2, 4, 6, 7, 5, 0, 3)]
    src = tmp_path / "src.bin"
    src_body = _body(299, BLOB // 2)
    src.write_bytes(src_body.tobytes())
    before = os.stat(src)
    with _engine(cas) as eng:
        eng.set_disk_limit(1 << 50)
        assert eng.verify(digs) == [demodel_b200.DM_OK] * N       # a scrub does not reorder the tier
        st, dig = eng.import_files([str(src)], link=True)[0]
        assert st == demodel_b200.DM_OK and dig == _sha(src_body)
        assert _read_all(eng, dig) == src_body.tobytes()          # a use: its recency stays in memory
        after = os.stat(src)
        assert after.st_mtime_ns == before.st_mtime_ns and after.st_ino == before.st_ino
        assert src.read_bytes() == src_body.tobytes()
        _evict_one_at_a_time(eng, cas, order[:4])
        _check_tier(eng, cas)


def test_hbm_engine_spills_under_the_limit(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(300 + i, BLOB) for i in range(N)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(1 << 50)
        first = _ingest(eng, bodies[0])
        one = eng.disk_usage()["used_bytes"]
        limit = 3 * one + one // 2                                 # room for three
        eng.set_disk_limit(limit)
        digs = [first] + [_ingest(eng, b) for b in bodies[1:]]
        u = eng.disk_usage()
        assert u["used_bytes"] <= limit and u["used_bytes"] == _walk(cas)
        on_disk = _present(cas, digs)
        assert on_disk == [False] * (N - 3) + [True] * 3          # HBM LRU order among HBM-resident blobs
        for d, b in zip(digs, bodies):                             # still served from HBM
            assert _read_all(eng, d) == b.tobytes()
        for d, there in zip(digs, on_disk):
            assert eng.cache_evict(d)
            if not there:
                assert eng.cache_contains(d) is None               # nothing to fall back to
        big = _body(399, 4 * one)                                  # its spill cannot fit at all
        sid = eng.stream_open(_sha(big), big.nbytes)
        eng.stream_write(sid, big)
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.stream_finish(sid)
        assert ei.value.code == demodel_b200.DM_EIO                # DM_F_DISK_SYNC: as after a failed spill
        assert eng.disk_usage()["refused"] == u["refused"] + 1
        assert _read_all(eng, _sha(big)) == big.tobytes()
        assert eng.cache_evict(_sha(big)) and eng.cache_contains(_sha(big)) is None
        _check_tier(eng, cas)


def test_disk_direct_body_over_the_limit_is_verified_not_cached(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    old = [_body(400 + i, BLOB) for i in range(3)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(1 << 50)
        old_digs = _disk_only(eng, old)
    one = _entry_bytes(cas, old_digs[0])
    with _engine(cas, hbm=SMALL_ARENA, flags=_lib.DM_F_DISK_DIRECT) as eng:
        limit = 3 * one + 4096
        eng.set_disk_limit(limit)
        huge = _body(410, limit + SLAB)
        seen = []
        sid = eng.stream_open(_sha(huge), huge.nbytes)
        for off in range(0, huge.nbytes, SLAB // 2):
            eng.stream_write(sid, huge[off:off + SLAB // 2])
            seen += _incoming(cas)
        dig, ok = eng.stream_finish(sid)
        assert ok and dig == _sha(huge) and not seen and not _incoming(cas)
        assert eng.cache_contains(dig) is None
        assert eng.disk_usage()["refused"] == 1
        assert all(_present(cas, old_digs))
        fits = _body(411, 2 * BLOB + 4096)                         # larger than the arena, fits the limit
        dig = _ingest(eng, fits)
        assert _read_all(eng, dig) == fits.tobytes()
        assert _present(cas, old_digs)[:2] == [False, False]       # the two oldest made its room
        assert eng.disk_usage()["used_bytes"] <= limit
        _check_tier(eng, cas)


def test_unknown_size_over_the_limit(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    with _engine(cas, flags=_lib.DM_F_NO_HBM_CAS | _lib.DM_F_DISK_DIRECT) as eng:
        eng.set_disk_limit(2 * BLOB)
        body = _body(500, 3 * BLOB + 123)
        dig = _ingest(eng, body, size_hint=False)
        assert dig == _sha(body) and eng.cache_contains(dig) is None and not _incoming(cas)
        assert eng.disk_usage()["refused"] == 1
        small = _body(501, BLOB // 2)
        dig = _ingest(eng, small, size_hint=False)                 # fits: cached
        assert _read_all(eng, dig) == small.tobytes()
        _check_tier(eng, cas)


def test_open_reader_pins_its_blob(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(600 + i, BLOB) for i in range(4)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(1 << 50)
        a, b = _disk_only(eng, bodies[:2])
        one = _entry_bytes(cas, a)
        eng.set_disk_limit(2 * one + 1024)
        rid, size = eng.cache_open(a)                              # a: open, then b becomes the most recent
        assert _read_all(eng, b) == bodies[1].tobytes()
        c = _ingest(eng, bodies[2])                                # its spill needs a's or b's room: a is pinned
        assert _present(cas, [a, b, c]) == [True, False, True]
        got = bytearray()
        while len(got) < size:
            got += eng.cache_read(rid, len(got), min(1 << 18, size - len(got)))
        assert bytes(got) == bodies[0].tobytes()
        eng.cache_close(rid)
        assert eng.cache_evict(c)
        d = _ingest(eng, bodies[3])                                # a is the least recent now
        assert _present(cas, [a, c, d]) == [False, True, True]
        _check_tier(eng, cas)


def test_import_past_the_room(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    srcs = []
    for i, n in enumerate((BLOB // 2, 3 * BLOB, 4 * BLOB)):
        p = tmp_path / f"src{i}.bin"
        p.write_bytes(_body(700 + i, n).tobytes())
        srcs.append(p)
    before = [(os.stat(p).st_ino, p.read_bytes()) for p in srcs]
    with _engine(cas) as eng:
        eng.set_disk_limit(2 * BLOB)
        res = eng.import_files([str(p) for p in srcs]) + eng.import_files([str(srcs[2])], link=True)
        assert [r[0] for r in res] == [demodel_b200.DM_OK, demodel_b200.DM_ENOMEM, demodel_b200.DM_ENOMEM,
                                       demodel_b200.DM_ENOMEM]
        assert res[0][1] == hashlib.sha256(before[0][1]).digest()
        assert [(os.stat(p).st_ino, p.read_bytes()) for p in srcs] == before
        assert not _incoming(cas)
        assert eng.disk_usage()["refused"] == 3
        _check_tier(eng, cas)


def test_saved_downloads_are_counted_and_evicted(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    body = _body(800, 2 * BLOB)
    with _engine(cas) as eng:
        eng.set_disk_limit(1 << 50)
        sid = eng.stream_open(_sha(body), body.nbytes)
        eng.stream_write(sid, body[:BLOB])
        assert eng.stream_suspend(sid) == BLOB
        u = eng.disk_usage()
        assert u["partial_bytes"] >= BLOB and u["used_bytes"] == _walk(cas)
        eng.set_disk_limit(1)
        assert eng.disk_usage()["partial_bytes"] == 0 and eng.stats()["suspended"] == 0
        assert eng.stream_resume_saved(_sha(body), body.nbytes) is None
        _check_tier(eng, cas)
    with _engine(cas, hbm=SMALL_ARENA, flags=_lib.DM_F_DISK_DIRECT) as eng:
        eng.set_disk_limit(1 << 50)
        big = _body(801, 3 * BLOB)
        sid = eng.stream_open(_sha(big), big.nbytes)
        eng.stream_write(sid, big[:BLOB])
        assert eng.stream_suspend(sid) == BLOB
        assert eng.disk_usage()["partial_bytes"] >= BLOB
        sid, off = eng.stream_resume_saved(_sha(big), big.nbytes)
        assert off == BLOB
        eng.set_disk_limit(1)                                      # the resumed stream's file is live: not a victim
        assert len(_incoming(cas)) == 1
        eng.stream_write_at(sid, off, big[off:])
        dig, ok = eng.stream_finish(sid)                           # no room at publish: verified, not cached
        assert ok and dig == _sha(big) and eng.cache_contains(dig) is None and not _incoming(cas)
        _check_tier(eng, cas)


def test_resume_in_progress_pins_its_saved_download(tmp_path):
    """While dm_stream_resume_saved loads a saved download back, other threads keep lowering the limit to one byte:
    the download is either evicted before the resume takes it (DM_ENOENT) or resumed whole, never lost half way."""
    cas = str(tmp_path / "cas")
    body = _body(850, 8 * BLOB)
    saved = 6 * BLOB
    resumed = 0
    with _engine(cas) as eng:
        eng.set_disk_limit(1 << 50)
        for delay in (0.0, 0.0005, 0.001, 0.002, 0.005, 0.02):
            sid = eng.stream_open(_sha(body), body.nbytes)
            eng.stream_write(sid, body[:saved])
            assert eng.stream_suspend(sid) == saved
            stop = threading.Event()

            def squeeze():
                time.sleep(delay)                              # the resume starts first, and pins, at some delays
                while not stop.is_set():
                    eng.set_disk_limit(1)
                    eng.set_disk_limit(1 << 50)

            th = threading.Thread(target=squeeze)
            th.start()
            try:
                got = eng.stream_resume_saved(_sha(body), body.nbytes)
            finally:
                stop.set()
                th.join()
            if got is None:
                continue
            sid, off = got
            assert off == saved
            eng.stream_write_at(sid, off, body[off:])
            dig, ok = eng.stream_finish(sid)
            assert ok and dig == _sha(body)
            assert _read_all(eng, dig) == body.tobytes()
            resumed += 1
        assert eng.stats()["suspended"] == 0
        _check_tier(eng, cas)
    print("resumed", resumed, "of 6")


def test_limit_one_empties_and_zero_turns_off(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(900 + i, BLOB // 4 + i) for i in range(N)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        assert eng.disk_usage() == dict(limit_bytes=0, used_bytes=0, blob_files=0, blob_bytes=0, staging_bytes=0,
                                        partial_bytes=0, evicted_files=0, evicted_bytes=0, refused=0)
        digs = _disk_only(eng, bodies)
        eng.set_disk_limit(1 << 50)
        total = _walk(cas)
        assert eng.disk_usage()["used_bytes"] == total and eng.disk_usage()["blob_files"] == N
        rid, _ = eng.cache_open(digs[2])                           # pinned through it all
        eng.set_disk_limit(1)
        u = eng.disk_usage()
        assert _present(cas, digs) == [i == 2 for i in range(N)]
        assert u["evicted_files"] == N - 1 and u["used_bytes"] == _walk(cas) > 1
        eng.cache_close(rid)
        eng.set_disk_limit(0)
        u = eng.disk_usage()
        assert u["limit_bytes"] == 0 and u["used_bytes"] == 0 and u["evicted_files"] == N - 1
        more = _ingest(eng, _body(999, BLOB))                      # no limit: nothing is evicted any more
        assert all(_present(cas, [digs[2], more]))
        _check_tier(eng, cas)


def test_errors(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    with _engine(None) as eng:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.set_disk_limit(1 << 30)
        assert ei.value.code == demodel_b200.DM_ESTATE
    with _engine(str(tmp_path / "cas")) as eng:
        u = _lib.DmDiskUsage()
        u.struct_size = C.sizeof(_lib.DmDiskUsage) - 8
        assert eng._lib.dm_cache_disk_usage(eng._h, C.byref(u)) == demodel_b200.DM_EINVAL
        assert eng._lib.dm_cache_set_disk_limit(None, 1) == demodel_b200.DM_EINVAL


def test_concurrent_placements_stay_under_the_limit(tmp_path):
    import demodel_b200
    from demodel_b200 import _lib
    cas = str(tmp_path / "cas")
    bodies = [_body(1000 + i, BLOB // 2 + 64 * i) for i in range(4 * N)]
    with _engine(cas, flags=_lib.DM_F_DISK_SYNC) as eng:
        eng.set_disk_limit(4 * BLOB)
        errs = []

        def worker(k):
            try:
                for b in bodies[k::4]:
                    d = _ingest(eng, b)
                    assert _read_all(eng, d) == b.tobytes()
                    eng.cache_evict(d)
                    got = eng.cache_open(d)
                    if got is not None:
                        eng.cache_close(got[0])
            except Exception as e:                                  # noqa: BLE001 - reported below
                errs.append(e)

        th = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        assert eng.disk_usage()["used_bytes"] <= 4 * BLOB
        _check_tier(eng, cas)
        st = eng.stats()
        assert st["open_readers"] == 0 and st["ring_slabs_free"] == st["ring_slabs_total"]
