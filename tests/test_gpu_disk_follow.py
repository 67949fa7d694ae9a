"""Followers of disk-backed bodies (dm_cache_follow on a DM_F_DISK_DIRECT stream): a second client reads a body that
another connection is still writing into <cas_dir>/incoming/, served from the body's file as its writes complete, and
becomes an ordinary disk-tier reader once the GPU's verdict is in.  The GPU hashes each body once, however many
clients read it.  Bodies come from the oracle's counter-based generator; what every follower returns is compared with
the source and with hashlib.

Sizes are module constants so that tests/test_disk_follow_host.py can run the same tests over the fake CUDA runtime with
a small ring and arena."""
import hashlib
import os
import random
import threading
import time

import pytest

from tests import _oracle

pytestmark = pytest.mark.gpu

ARENA = 8 << 20             # HBM arena; every body here is larger
RING = 32 << 20
SLAB = 1 << 20
BODY = (24 << 20) + 4321    # one followed body
WRITE = 64 << 10            # the owner's pieces
READ = 32 << 10             # the followers' pieces (io.Copy)
SEED = 0xF0110


def _flags(disk_only):
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    return DM_F_DISK_DIRECT | (DM_F_NO_HBM_CAS if disk_only else 0)


def _engine(cas, disk_only=False, flags=None):
    import demodel_b200
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, slab_bytes=SLAB, cas_dir=cas,
                               flags=_flags(disk_only) if flags is None else flags)


def _body(k, n=None):
    return _oracle.load().blob(SEED, k, 0, BODY if n is None else n)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _incoming(cas):
    d = os.path.join(cas, "incoming")
    return os.listdir(d) if os.path.isdir(d) else []


def _clean(eng, cas):
    for _ in range(500):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == 65536
                and st["open_streams"] == 0 and st["open_readers"] == 0 and not _incoming(cas)):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}, incoming/ {_incoming(cas)}")


class Follower(threading.Thread):
    """Reads a followed body front to back in READ-byte pieces until EOF (an empty read) or an error, the way an HTTP
    response body is copied out."""

    def __init__(self, eng, rid, hint, want, start=0):
        super().__init__(daemon=True)
        self.eng, self.rid, self.hint, self.want, self.pos = eng, rid, hint, want, start
        self.got = bytearray()
        self.err = None
        self.cached_at_eof = None           # dm_cache_contains right after the EOF read returned
        self.on_first = None                # an Event set once the first bytes are in

    def run(self):
        import demodel_b200
        try:
            while True:
                piece = self.eng.cache_read(self.rid, self.pos, READ)
                if not piece:
                    self.cached_at_eof = self.eng.cache_contains(self.want)
                    return
                self.got += piece
                self.pos += len(piece)
                if self.on_first:
                    self.on_first.set()
        except demodel_b200.DmError as ex:
            self.err = ex


def _follow(eng, dig, n, start=0):
    out = []
    for _ in range(n):
        got = eng.cache_follow(dig)
        assert got is not None
        out.append(Follower(eng, *got, dig, start))
    return out


def _write(eng, sid, body, start=0, end=None):
    end = body.nbytes if end is None else end
    for off in range(start, end, WRITE):
        eng.stream_write(sid, body[off:min(end, off + WRITE)])


@pytest.mark.parametrize("disk_only", [False, True])
def test_sequential_followers_get_the_body_and_wait_for_the_verdict(tmp_path, disk_only):
    """1, then 8 followers attach before the first byte and read 32 KiB pieces while the owner writes 64 KiB pieces.
    Every follower gets the exact body; its EOF read returns once the blob is in the tier; it then serves random
    offsets as a cache reader with the published sidecar; the GPU hashed the body once."""
    cas = str(tmp_path / "cas")
    eng = _engine(cas, disk_only)
    try:
        for k, n in enumerate((1, 8)):
            body = _body(k)
            want = _sha(body)
            assert eng.cache_follow(want) is None                       # nothing in flight
            hashed0 = eng.stats()["bytes_hashed"]
            served0 = eng.stats()["bytes_served"]
            sid = eng.stream_open(want, body.nbytes)
            fs = _follow(eng, want, n)
            assert all(f.hint == body.nbytes for f in fs)
            assert eng.stats()["open_readers"] == n
            for f in fs:
                f.start()
            _write(eng, sid, body)
            dig, ok = eng.stream_finish(sid)
            assert ok and dig == want
            for f in fs:
                f.join(120)
                assert not f.is_alive() and f.err is None
                assert bytes(f.got) == body.tobytes() and _sha(body) == hashlib.sha256(f.got).digest()
                assert f.cached_at_eof == body.nbytes                   # the EOF read came after the verdict
            st = eng.stats()
            assert st["bytes_hashed"] - hashed0 == body.nbytes          # one hash, however many readers
            assert st["bytes_served"] - served0 >= n * body.nbytes
            rng = random.Random(k)
            for f in fs:
                for _ in range(8):
                    off = rng.randrange(body.nbytes)
                    ln = rng.randrange(1, 100000)
                    assert eng.cache_read(f.rid, off, ln) == body[off:off + ln].tobytes()
                assert eng.cache_read(f.rid, body.nbytes, 10) == b""
                meta = eng.cache_meta(f.rid)
                assert meta["digest"] == "sha256:" + want.hex() and meta["size"] == body.nbytes
                eng.cache_close(f.rid)
            with open(_blob_file(cas, want), "rb") as fh:
                assert hashlib.sha256(fh.read()).digest() == want
        _clean(eng, cas)
    finally:
        eng.close()


def test_range_parts_are_served_as_they_land(tmp_path):
    """Four parts written out of order (last, second, third, first).  A follower inside the last part is served while
    the first part is not written yet; a follower at offset 0 waits for the prefix and gets the whole body."""
    cas = str(tmp_path / "cas")
    eng = _engine(cas)
    try:
        body = _body(10)
        want = _sha(body)
        q = (body.nbytes // 4) // SLAB * SLAB
        bounds = [0, q, 2 * q, 3 * q, body.nbytes]
        sid = eng.stream_open(want, body.nbytes)
        inner = bounds[3] + 100
        late = threading.Event()
        f0 = _follow(eng, want, 1)[0]
        f3 = _follow(eng, want, 1, start=inner)[0]
        f3.on_first = late
        f0.start()
        f3.start()

        def part(i):
            for off in range(bounds[i], bounds[i + 1], WRITE):
                eng.stream_write_at(sid, off, body[off:min(bounds[i + 1], off + WRITE)])

        part(3)
        assert late.wait(60), "a follower inside a written part was not served before the prefix"
        assert not f0.got                                                # offset 0: nothing written there yet
        part(1)
        part(2)
        part(0)
        dig, ok = eng.stream_finish(sid)
        assert ok and dig == want
        for f in (f0, f3):
            f.join(120)
            assert f.err is None
        assert bytes(f0.got) == body.tobytes()
        assert bytes(f3.got) == body[inner:].tobytes()
        for f in (f0, f3):
            eng.cache_close(f.rid)
        _clean(eng, cas)
    finally:
        eng.close()


def test_unknown_size_on_a_disk_only_engine(tmp_path):
    """A body opened without Content-Length: the follower is told 0 (unknown) and learns the size at EOF."""
    import demodel_b200
    cas = str(tmp_path / "cas")
    eng = _engine(cas, disk_only=True)
    try:
        body = _body(20, BODY - 777)
        want = _sha(body)
        sid = eng.stream_open(want, 0)
        (f,) = _follow(eng, want, 1)
        assert f.hint == 0
        f.start()
        _write(eng, sid, body)
        assert eng.stream_finish(sid) == (want, True)
        f.join(120)
        assert f.err is None and bytes(f.got) == body.tobytes()
        assert eng.cache_read(f.rid, body.nbytes, 10) == b""
        with pytest.raises(demodel_b200.DmError) as ex:
            eng.cache_read(f.rid, body.nbytes + 1, 10)
        assert ex.value.code == demodel_b200.DM_ERANGE
        assert eng.cache_meta(f.rid)["size"] == body.nbytes
        eng.cache_close(f.rid)
        _clean(eng, cas)
    finally:
        eng.close()


@pytest.mark.parametrize("mode", ["abort", "corrupt", "suspend"])
def test_failures_end_in_estate_never_wrong_bytes(tmp_path, mode):
    """An abort mid-body, a corrupted byte and a suspend each end the follower's reads with DM_ESTATE and a detail text
    naming the cause; every byte it got before is a byte the owner wrote.  After a suspend, dm_stream_resume_saved
    makes the body followable again from byte 0: a new follower reads the saved prefix and the rest to the verified
    end."""
    import demodel_b200
    cas = str(tmp_path / "cas")
    eng = _engine(cas)
    try:
        body = _body(30)
        want = _sha(body)
        sent = body.copy()
        half = body.nbytes // 2
        if mode == "corrupt":
            sent[half + 5] ^= 1
        sid = eng.stream_open(want, body.nbytes)
        (f,) = _follow(eng, want, 1)
        seen = threading.Event()
        f.on_first = seen
        f.start()
        _write(eng, sid, sent, 0, half)
        assert seen.wait(60)
        resume_from = None
        if mode == "abort":
            eng.stream_abort(sid)
        elif mode == "suspend":
            resume_from = eng.stream_suspend(sid)
        else:
            _write(eng, sid, sent, half)
            dig, ok = eng.stream_finish(sid)
            assert not ok
        f.join(120)
        assert not f.is_alive()
        assert f.err is not None and f.err.code == demodel_b200.DM_ESTATE
        assert bytes(f.got) == sent[:len(f.got)].tobytes()
        text = eng.error_detail(f.rid)
        assert {"abort": "aborted", "corrupt": "verification", "suspend": "suspended"}[mode] in text, text
        with pytest.raises(demodel_b200.DmError):
            eng.cache_read(f.rid, len(f.got), READ)
        eng.cache_close(f.rid)
        assert eng.cache_follow(want) is None
        if mode == "suspend":
            sid, start = eng.stream_resume_saved(want, body.nbytes)
            assert start == resume_from and 0 < start <= half
            (g,) = _follow(eng, want, 1)
            g.start()
            _write(eng, sid, body, start)
            assert eng.stream_finish(sid) == (want, True)
            g.join(120)
            assert g.err is None and bytes(g.got) == body.tobytes()
            eng.cache_close(g.rid)
        _clean(eng, cas)
    finally:
        eng.close()


def test_a_follower_past_eof_pins_the_blob(tmp_path):
    """A follower that has read to EOF holds the tier file like a dm_cache_open reader: a limit of 1 byte evicts the
    blob only after dm_cache_close."""
    cas = str(tmp_path / "cas")
    eng = _engine(cas)
    try:
        body = _body(40)
        want = _sha(body)
        sid = eng.stream_open(want, body.nbytes)
        (f,) = _follow(eng, want, 1)
        f.start()
        _write(eng, sid, body)
        assert eng.stream_finish(sid) == (want, True)
        f.join(120)
        assert f.err is None and bytes(f.got) == body.tobytes()
        eng.set_disk_limit(1)
        assert os.path.exists(_blob_file(cas, want))
        assert eng.cache_read(f.rid, 0, 1000) == body[:1000].tobytes()
        eng.cache_close(f.rid)
        eng.set_disk_limit(1)
        assert not os.path.exists(_blob_file(cas, want))
        assert eng.disk_usage()["used_bytes"] == 0
        _clean(eng, cas)
    finally:
        eng.close()


def test_unknown_size_refused_at_publish_is_read_to_the_end(tmp_path):
    """An unknown-size body whose final size does not fit under the limit is verified and not cached; its follower still
    reads it to the end from its own descriptor."""
    cas = str(tmp_path / "cas")
    eng = _engine(cas, disk_only=True)
    try:
        eng.set_disk_limit(BODY // 2)
        body = _body(50)
        want = _sha(body)
        refused0 = eng.disk_usage()["refused"]
        sid = eng.stream_open(want, 0)
        (f,) = _follow(eng, want, 1)
        f.start()
        _write(eng, sid, body)
        assert eng.stream_finish(sid) == (want, True)
        f.join(120)
        assert f.err is None and bytes(f.got) == body.tobytes()
        assert f.cached_at_eof is None
        assert eng.disk_usage()["refused"] == refused0 + 1
        assert eng.cache_read(f.rid, 12345, 999) == body[12345:12345 + 999].tobytes()
        assert eng.cache_meta(f.rid)["digest"] == "sha256:" + want.hex()
        eng.cache_close(f.rid)
        assert eng.cache_contains(want) is None and not os.path.exists(_blob_file(cas, want))
        _clean(eng, cas)
    finally:
        eng.close()


def test_streams_that_retain_nothing_are_not_followable(tmp_path):
    """A verify-only stream (no DM_F_DISK_DIRECT) and a disk-backed open refused by the limit keep no bytes to serve:
    dm_cache_follow says DM_ENOENT, as for a digest nothing is ingesting."""
    from demodel_b200._lib import DM_F_NO_HBM_CAS
    body = _body(60, 3 * SLAB + 5)
    want = _sha(body)
    cas = str(tmp_path / "cas")
    for flags, limit in ((DM_F_NO_HBM_CAS, 0), (_flags(True), 1)):
        eng = _engine(cas, flags=flags)
        try:
            if limit:
                eng.set_disk_limit(limit)
            sid = eng.stream_open(want, body.nbytes)
            assert eng.cache_follow(want) is None
            _write(eng, sid, body)
            assert eng.stream_finish(sid) == (want, True)
            assert eng.cache_contains(want) is None
            _clean(eng, cas)
        finally:
            eng.close()
