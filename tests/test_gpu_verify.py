"""dm_cache_verify and dm_cache_list on the GPU: disk-tier files are hashed in place by the SHA-256 kernels, read back
through the ring by the disk threads (or, at most tiny_max bytes, through packs), without touching the HBM arena.
Every body is checked against hashlib over the same bytes.

Sizes are module constants so that tests/test_verify_host.py can run the same tests over the fake CUDA runtime with a
small ring and arena."""
import hashlib
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 512 << 20           # HBM arena of the checking engines
RING = 64 << 20
SLAB = 1 << 20
SMALL_ARENA = 16 << 20      # the arena a blob larger than it lives next to
MANY = 3000                 # tiny bodies (at most 8 KiB) in one call
MANY_BIG = 512              # ... and this many bodies of one slab
MANY_ARENA = 2 << 30        # the arena that caches them first
LIVE_BLOBS = 64             # multi-slab blobs checked while live writers stream
LIST_N = 40


def _tiny_max():
    return min(64 << 10, SLAB // 4)


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    kw.setdefault("ring_bytes", RING)
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, slab_bytes=SLAB, cas_dir=cas,
                               **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for off in range(0, body.nbytes, 1 << 20):
        eng.stream_write(sid, body[off:off + (1 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _populate(cas, bodies, **kw):
    """Cache the bodies through ordinary streams, then destroy the engine (its spills drain): all on disk only."""
    with _engine(cas, **kw) as eng:
        digs = [_ingest(eng, b) for b in bodies]
    for d, b in zip(digs, bodies):
        assert os.path.getsize(_blob_file(cas, d)) == b.nbytes
    return digs


def _flip(path, at):
    with open(path, "r+b") as f:
        f.seek(at)
        b = f.read(1)
        f.seek(at)
        f.write(bytes([b[0] ^ 0x01]))


def _hashes_to_name(cas, dig):
    with open(_blob_file(cas, dig), "rb") as f:
        return hashlib.sha256(f.read()).digest() == dig


def _on_disk_only(eng, dig):
    import demodel_b200
    rid, _ = eng.cache_open(dig)
    try:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.cache_device_extents(rid)
        assert ei.value.code == demodel_b200.DM_ESTATE
    finally:
        eng.cache_close(rid)


def _read_all(eng, rid, size):
    got = bytearray()
    while len(got) < size:
        part = eng.cache_read(rid, len(got), min(4 << 20, size - len(got)))
        assert part
        got += part
    return bytes(got)


def _clean(eng, max_streams=65536):
    import time
    for _ in range(400):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == 0):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _wait_for_verified_file(cas, dig):
    import time
    for _ in range(500):
        try:
            if _hashes_to_name(cas, dig) and os.path.exists(_blob_file(cas, dig) + ".meta"):
                return
        except FileNotFoundError:
            pass
        time.sleep(0.01)
    raise AssertionError("the disk tier never got a copy that hashes to its name")


def test_good_blobs_at_the_sizes_that_matter(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    t = _tiny_max()
    sizes = [0, 1, 63, 64, 65, 8192, t, t + 1, SLAB - 1, SLAB, SLAB + 1, 3 * SLAB + 17]
    bodies = [_body(100 + i, n) for i, n in enumerate(sizes)]
    digs = _populate(cas, bodies)
    inodes = [os.stat(_blob_file(cas, d)).st_ino for d in digs]
    with _engine(cas) as eng:
        st0 = eng.stats()
        assert eng.verify(digs) == [DM_OK] * len(digs)
        st = eng.stats()
        assert st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert st["bytes_hashed"] - st0["bytes_hashed"] == sum(sizes)
        assert st["h2d_bytes"] - st0["h2d_bytes"] == sum(sizes)
        assert st["blobs_committed"] == st0["blobs_committed"] and st["blobs_mismatched"] == st0["blobs_mismatched"]
        assert st["kernel_launches"] > st0["kernel_launches"] and st["d2h_bytes"] == st0["d2h_bytes"]
        for d, b in zip(digs, bodies):
            _on_disk_only(eng, d)
            assert eng.fetch(d, chunk=4 << 20) == b.tobytes()
        assert eng.verify([]) == []
        _clean(eng)
    assert [os.stat(_blob_file(cas, d)).st_ino for d in digs] == inodes


def test_corruption_at_the_edges(tmp_path):
    from demodel_b200 import DM_ECORRUPT, DM_OK
    cas = str(tmp_path / "cas")
    n = 3 * SLAB + 100
    bodies = [_body(200 + i, n) for i in range(7)] + [_body(210, 5000), _body(211, 5000), _body(212, n)]
    digs = _populate(cas, bodies)
    first, last, before, after, trunc, longer, lies, tiny, tiny_clean, clean = digs
    _flip(_blob_file(cas, first), 10)
    _flip(_blob_file(cas, last), n - 3)
    _flip(_blob_file(cas, before), SLAB - 1)
    _flip(_blob_file(cas, after), SLAB)
    os.truncate(_blob_file(cas, trunc), n - 1)
    with open(_blob_file(cas, longer), "ab") as f:
        f.write(b"x")
    meta = _blob_file(cas, lies) + ".meta"
    with open(meta) as f:
        text = f.read()
    assert f'"size":{n},' in text
    with open(meta, "w") as f:
        f.write(text.replace(f'"size":{n},', f'"size":{n + 1},'))
    _flip(_blob_file(cas, tiny), 4999)
    bad = [first, last, before, after, trunc, longer, lies, tiny]
    with _engine(cas) as eng:
        st0 = eng.stats()
        assert eng.verify(digs) == [DM_ECORRUPT] * len(bad) + [DM_OK, DM_OK]
        st = eng.stats()
        assert st["blobs_mismatched"] == st0["blobs_mismatched"] and st["hbm_cas_used"] == st0["hbm_cas_used"]
        for d in bad:
            assert not os.path.exists(_blob_file(cas, d)) and not os.path.exists(_blob_file(cas, d) + ".meta")
            assert eng.cache_contains(d) is None and eng.cache_open(d) is None
        for d, b in ((tiny_clean, bodies[8]), (clean, bodies[9])):
            assert _hashes_to_name(cas, d) and eng.fetch(d, chunk=4 << 20) == b.tobytes()
        _clean(eng)


def test_blob_larger_than_the_arena(tmp_path):
    from demodel_b200 import DM_ECORRUPT, DM_ENOMEM, DM_OK
    from demodel_b200._lib import DM_F_DISK_DIRECT
    cas = str(tmp_path / "cas")
    body = _body(300, SMALL_ARENA + 12345)
    with _engine(cas, hbm=SMALL_ARENA, flags=DM_F_DISK_DIRECT) as eng:       # cached on disk by a disk-backed stream
        dig = _ingest(eng, body)
        assert eng.verify([dig]) == [DM_OK]                                   # with the flag
    with _engine(cas, hbm=SMALL_ARENA) as eng:                                # and without it
        st0 = eng.stats()
        assert eng.verify([dig]) == [DM_OK]
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes and st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert eng.promote([dig]) == [DM_ENOMEM]
        _clean(eng)
    _flip(_blob_file(cas, dig), body.nbytes // 2)
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        assert eng.verify([dig]) == [DM_ECORRUPT]
        assert not os.path.exists(_blob_file(cas, dig)) and eng.cache_contains(dig) is None
        _clean(eng)


def test_disk_only_engine(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_ECORRUPT, DM_ENOENT, DM_ESTATE, DM_OK
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    bodies = [_body(400 + i, n) for i, n in enumerate([0, 100, 70000, 2 * SLAB + 3])]
    flags = DM_F_NO_HBM_CAS | DM_F_DISK_DIRECT
    with _engine(cas, flags=flags) as eng:
        digs = [_ingest(eng, b) for b in bodies]
    _flip(_blob_file(cas, digs[2]), 7)
    missing = hashlib.sha256(b"never cached").digest()
    with _engine(cas, flags=flags) as eng:
        assert eng.verify(digs + [missing]) == [DM_OK, DM_OK, DM_ECORRUPT, DM_OK, DM_ENOENT]
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.promote(digs)
        assert ei.value.code == DM_ESTATE
        assert eng.fetch(digs[3], chunk=4 << 20) == bodies[3].tobytes()
        _clean(eng)


def test_blob_in_hbm_with_a_damaged_disk_copy(tmp_path):
    from demodel_b200 import DM_ECORRUPT
    cas = str(tmp_path / "cas")
    body = _body(500, 2 * SLAB + 11)
    with _engine(cas) as eng:
        dig = _ingest(eng, body)
        _wait_for_verified_file(cas, dig)
        _flip(_blob_file(cas, dig), 12345)
        used = eng.stats()["hbm_cas_used"]
        assert eng.verify([dig]) == [DM_ECORRUPT]
        assert eng.stats()["hbm_cas_used"] == used
        rid, size = eng.cache_open(dig)                                        # the HBM copy is still served
        assert size == body.nbytes and _read_all(eng, rid, size) == body.tobytes()
        eng.cache_close(rid)
        _wait_for_verified_file(cas, dig)                                      # written out again from HBM
        _clean(eng)
    with _engine(cas) as eng:
        assert eng.fetch(dig, chunk=4 << 20) == body.tobytes()
        _clean(eng)


def test_engine_without_a_disk_tier(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_ENOENT, DM_OK
    body = _body(600, 1000)
    missing = hashlib.sha256(b"never cached").digest()
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, slab_bytes=SLAB) as eng:
        dig = _ingest(eng, body)
        st0 = eng.stats()
        assert eng.verify([dig, missing, dig]) == [DM_OK, DM_ENOENT, DM_OK]
        assert eng.stats()["bytes_hashed"] == st0["bytes_hashed"]
        assert eng.list() == [] and eng.list(after=dig, cap=7) == []
        _clean(eng)


def test_many_blobs_share_launches(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    rng = np.random.default_rng(700)
    sizes = rng.integers(1, 8192, MANY)
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    host = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    big = [_body(701 + i, SLAB) for i in range(MANY_BIG)]
    with _engine(cas, hbm=MANY_ARENA) as eng:
        tiny, ok, _ = eng.proxy_drive(host, offsets, concurrency=64, nthreads=4)
        assert all(ok)
        large = [_ingest(eng, b) for b in big]
    with _engine(cas) as eng:
        st0 = eng.stats()
        assert eng.verify(tiny) == [DM_OK] * MANY
        st = eng.stats()
        assert st["kernel_launches"] - st0["kernel_launches"] < 300            # the chains went out together
        assert st["bytes_hashed"] - st0["bytes_hashed"] == int(offsets[-1])
        everything = tiny + large + tiny[:100] + large[:10]                       # duplicates are checked once
        st0 = eng.stats()
        assert eng.verify(everything) == [DM_OK] * len(everything)
        st = eng.stats()
        want = int(offsets[-1]) + SLAB * MANY_BIG
        assert st["bytes_hashed"] - st0["bytes_hashed"] == want
        assert st["h2d_bytes"] - st0["h2d_bytes"] == want
        assert st["hbm_cas_used"] == st0["hbm_cas_used"] == 0
        _clean(eng)


def test_live_writers_finish_while_a_large_verify_runs(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(800 + i, 3 * SLAB + 5 + i) for i in range(LIVE_BLOBS)]
    digs = _populate(cas, bodies)
    with _engine(cas, ring_bytes=16 * SLAB) as eng:
        out = {}
        t = threading.Thread(target=lambda: out.setdefault("st", eng.verify(digs)))
        done = []
        errors = []

        def writer(k):
            try:
                i = 0
                while t.is_alive() or i == 0:
                    b = _body(900 + 1000 * k + i, 2 * SLAB + 7 + k)
                    sid = eng.stream_open(_sha(b), b.nbytes)
                    for off in range(0, b.nbytes, 32 << 10):
                        eng.stream_write(sid, b[off:off + (32 << 10)])
                    dig, ok = eng.stream_finish(sid)
                    assert ok and dig == _sha(b)
                    done.append(dig)
                    i += 1
            except Exception as ex:                                            # reported by the main thread
                errors.append(ex)
        t.start()
        ws = [threading.Thread(target=writer, args=(k,)) for k in range(8)]
        for w in ws:
            w.start()
        t.join()
        for w in ws:
            w.join()
        assert not errors, errors
        assert out["st"] == [DM_OK] * LIVE_BLOBS
        assert len(done) >= 8
        _clean(eng)


def test_verify_races_a_stream_publishing_the_same_digest(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1000, 4 * SLAB + 3), _body(1001, 3000)]
    digs = _populate(cas, bodies)
    for _ in range(3):
        # a restarted engine does not know the files: each ingest publishes a fresh blob, whose spill renames a new
        # file over the one the check may be reading
        with _engine(cas) as eng:
            out = {}
            t = threading.Thread(target=lambda: out.setdefault("st", eng.verify(digs)))
            t.start()
            for d, b in zip(digs, bodies):
                assert _ingest(eng, b) == d
            t.join()
            assert out["st"] == [DM_OK, DM_OK]
            _clean(eng)
        for d in digs:
            assert _hashes_to_name(cas, d) and os.path.exists(_blob_file(cas, d) + ".meta")


def test_verify_races_a_promotion_of_an_overlapping_set(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1100 + i, (i + 1) * 300001) for i in range(8)]
    digs = _populate(cas, bodies)
    with _engine(cas) as eng:
        res = [None, None]

        def run(k, fn, subset):
            res[k] = fn(subset)
        th = [threading.Thread(target=run, args=(0, eng.verify, digs[:6])),
              threading.Thread(target=run, args=(1, eng.promote, digs[2:][::-1]))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert res == [[DM_OK] * 6, [DM_OK] * 6]
        assert eng.verify(digs) == [DM_OK] * 8
        for d, b in zip(digs, bodies):
            assert _hashes_to_name(cas, d) and eng.fetch(d, chunk=4 << 20) == b.tobytes()
        _clean(eng)


def test_the_last_free_stream_slot_stays_with_dm_stream_open(tmp_path):
    from demodel_b200 import DM_ENOMEM, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1200, 1000), _body(1201, 2 * SLAB)]
    digs = _populate(cas, bodies)
    with _engine(cas, max_streams=3) as eng:
        held = [eng.stream_open(None, 0) for _ in range(2)]
        assert eng.verify(digs) == [DM_ENOMEM, DM_ENOMEM]                     # one slot free: it is not taken
        last = eng.stream_open(None, 0)
        for s in held + [last]:
            eng.stream_abort(s)
        assert eng.verify(digs) == [DM_OK, DM_OK]
        for d in digs:
            assert _hashes_to_name(cas, d)
        _clean(eng, max_streams=3)


def test_list_pages_over_the_tier(tmp_path):
    cas = str(tmp_path / "cas")
    bodies = [_body(1300 + i, 100 + 37 * i) for i in range(LIST_N)]
    digs = _populate(cas, bodies)
    size_of = {d: b.nbytes for d, b in zip(digs, bodies)}
    # strays that must never be listed
    d0 = digs[0].hex()
    other = next(d for d in digs if d.hex()[:2] != d0[:2])
    stray_dir = os.path.join(cas, "blobs", "sha256", other.hex()[:2])
    strays = [_blob_file(cas, digs[0]) + ".part",
              os.path.join(os.path.dirname(_blob_file(cas, digs[0])), d0.upper()),
              os.path.join(stray_dir, hashlib.sha256(b"misplaced").hexdigest()),
              os.path.join(stray_dir, "notes.txt")]
    if hashlib.sha256(b"misplaced").hexdigest()[:2] == other.hex()[:2]:
        strays.pop(2)
    for p in strays:
        with open(p, "wb") as f:
            f.write(b"stray")
    with _engine(cas) as eng:
        got, after = [], None
        while True:
            page = eng.list(after=after, cap=7)
            assert len(page) <= 7
            got += page
            if len(page) < 7:
                break
            after = page[-1][0]
        assert [d for d, _ in got] == sorted(digs)
        assert all(size_of[d] == n for d, n in got)
        assert eng.list(after=max(digs)) == []
        assert eng.list(cap=0) == []
        _clean(eng)
    for p in strays:
        assert os.path.exists(p)
