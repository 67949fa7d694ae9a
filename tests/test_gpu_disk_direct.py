"""Disk-backed streams (DM_F_DISK_DIRECT) on the GPU: bodies larger than the HBM arena are written to
<cas_dir>/incoming/ as they arrive, hashed on the GPU from the bytes read back from that file, and the verified
file is renamed into the disk tier.  Digests are checked against hashlib; the published file, its sidecar and
what dm_cache_read serves are compared with the body byte for byte.

The arena is ARENA bytes and bodies are a few ARENA long, so every body here is over-arena (96-300 MiB on the GPU;
tests/test_disk_direct_host.py runs the same tests over the fake runtime with a smaller ARENA)."""
import hashlib
import json
import os
import random
import shutil
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 64 << 20
RING = 64 << 20


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _engine(cas, flags=None, hbm=None, **kw):
    import demodel_b200
    from demodel_b200._lib import DM_F_DISK_DIRECT
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, ring_bytes=RING, cas_dir=cas,
                               flags=DM_F_DISK_DIRECT if flags is None else flags, **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _write(eng, sid, body, chunk=1 << 20, start=0, end=None):
    end = body.nbytes if end is None else end
    for off in range(start, end, chunk):
        eng.stream_write(sid, body[off:min(end, off + chunk)])


def _read_all(eng, rid, size, piece=4 << 20):
    got = bytearray()
    while len(got) < size:
        part = eng.cache_read(rid, len(got), min(piece, size - len(got)))
        assert part
        got += part
    return bytes(got)


def _check_published(eng, cas, body, dig):
    path = _blob_file(cas, dig)
    with open(path, "rb") as f:
        assert f.read() == body.tobytes()
    meta = json.load(open(path + ".meta"))
    assert meta["digest"] == "sha256:" + dig.hex() and meta["size"] == body.nbytes
    rid, size = eng.cache_open(dig)
    try:
        assert size == body.nbytes and _read_all(eng, rid, size) == body.tobytes()
    finally:
        eng.cache_close(rid)
    assert os.listdir(os.path.join(cas, "incoming")) == []


def test_sequential_over_arena_body_is_cached_on_disk(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(1, ARENA + ARENA // 2 + 12345)
    want = hashlib.sha256(body.tobytes()).digest()
    with _engine(cas) as eng:
        st0 = eng.stats()
        sid = eng.stream_open(want, body.nbytes)
        eng.stream_set_meta(sid, "content-type", "application/octet-stream")
        _write(eng, sid, body)
        dig, ok = eng.stream_finish(sid)
        assert ok and dig == want
        assert os.path.exists(_blob_file(cas, dig))                    # in its final place when finish returns
        st = eng.stats()
        assert st["hbm_cas_used"] == st0["hbm_cas_used"]               # nothing of it went to HBM
        assert st["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes
        assert st["bytes_ingested"] - st0["bytes_ingested"] == body.nbytes
        assert st["blobs_committed"] - st0["blobs_committed"] == 1
        _check_published(eng, cas, body, dig)
        rid, _ = eng.cache_open(dig)
        assert eng.cache_meta(rid)["headers"]["content-type"] == "application/octet-stream"
        eng.cache_close(rid)
        assert st["open_streams"] == 0 and st["ring_slabs_free"] == st["ring_slabs_total"]


def test_parallel_range_parts_in_shuffled_order(tmp_path):
    cas = str(tmp_path / "cas")
    body = _body(2, 4 * ARENA + ARENA // 2 + 4097)
    want = hashlib.sha256(body.tobytes()).digest()
    cuts = sorted(random.Random(3).sample(range(1, body.nbytes), 15))
    parts = list(zip([0] + cuts, cuts + [body.nbytes]))
    random.Random(4).shuffle(parts)
    with _engine(cas) as eng:
        sid = eng.stream_open(want, body.nbytes)
        errors = []

        def part(lo, hi):
            try:
                for off in range(lo, hi, 1 << 20):
                    eng.stream_write_at(sid, off, body[off:min(hi, off + (1 << 20))])
            except Exception as ex:                                    # reported by the main thread
                errors.append(ex)
        th = [threading.Thread(target=part, args=p) for p in parts]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        dig, ok = eng.stream_finish(sid)
        assert ok and dig == want
        _check_published(eng, cas, body, dig)


def test_wrong_digest_and_abort_leave_nothing_behind(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(5, ARENA + ARENA // 2 + 1)
    want = hashlib.sha256(body.tobytes()).digest()
    with _engine(cas) as eng:
        st0 = eng.stats()
        dig, ok = eng.ingest(body, expect=bytes(32), chunk=1 << 20)
        assert not ok and dig == want
        assert eng.stats()["blobs_mismatched"] == st0["blobs_mismatched"] + 1
        assert not os.path.exists(_blob_file(cas, want)) and eng.cache_open(want) is None
        sid = eng.stream_open(want, body.nbytes)
        _write(eng, sid, body, end=body.nbytes // 2)
        eng.stream_abort(sid)
        with pytest.raises(demodel_b200.DmError):
            eng.stream_write(sid, body[:10])
        st = eng.stats()
        assert st["open_streams"] == 0 and st["ring_slabs_free"] == st["ring_slabs_total"]
        assert os.listdir(os.path.join(cas, "incoming")) == []
        assert not os.path.exists(os.path.join(cas, "blobs", "sha256", want.hex()[:2]))


def test_url_fetch_without_digest_hits_from_disk_also_after_a_restart(tmp_path):
    cas = str(tmp_path / "cas")
    url = "https://huggingface.co/org/big-model/resolve/main/model-00001-of-00002.safetensors"
    body = _body(6, ARENA + ARENA // 2 + 777)
    with _engine(cas) as e1:
        assert e1.proxy_request(url) is None
        dig, ok = e1.proxy_fetch(url, body, chunk=1 << 20)             # expect = NULL: digest learned by hashing
        assert ok and dig == hashlib.sha256(body.tobytes()).digest()
        rid, size = e1.proxy_request(url)
        assert _read_all(e1, rid, size) == body.tobytes()
        e1.cache_close(rid)
    with _engine(cas) as e2:                                           # restart over the same directory
        rid, size = e2.proxy_request(url)
        assert size == body.nbytes and _read_all(e2, rid, size) == body.tobytes()
        e2.cache_close(rid)


def _suspend_with_parts(eng, cas, body, want, head, islands):
    sid = eng.stream_open(want, body.nbytes)
    _write(eng, sid, body, end=head)
    for lo, hi in islands:
        eng.stream_write_at(sid, lo, body[lo:hi])
    (incoming,) = os.listdir(os.path.join(cas, "incoming"))
    ino = os.stat(os.path.join(cas, "incoming", incoming)).st_ino
    saved = eng.stream_suspend(sid)
    assert saved == head // 64 * 64                                   # the islands past the hole are not kept
    part = os.path.join(cas, "partial", want.hex() + ".part")
    assert os.stat(part).st_ino == ino and os.path.getsize(part) == saved      # renamed, not copied
    assert os.listdir(os.path.join(cas, "incoming")) == [] and eng.stats()["open_streams"] == 0
    return saved


@pytest.mark.parametrize("resume_on", ["disk", "hbm"])
def test_suspend_after_out_of_order_parts_then_resume_on_a_new_engine(tmp_path, resume_on):
    cas = str(tmp_path / "cas")
    body = _body(7, ARENA + ARENA // 2 + 999)
    want = hashlib.sha256(body.tobytes()).digest()
    head = ARENA // 2 + 12345
    islands = [(ARENA + 100, ARENA + 100 + (3 << 20)), (ARENA // 2 + 54321, ARENA // 2 + 54321 + 70001)]
    with _engine(cas) as e1:
        saved = _suspend_with_parts(e1, cas, body, want, head, islands)
        assert e1.stats()["suspended"] == 1
    # "disk": the same configuration; "hbm": no DM_F_DISK_DIRECT and an arena that now holds the blob
    kw = {} if resume_on == "disk" else {"flags": 0, "hbm": 4 * ARENA}
    with _engine(cas, **kw) as e2:
        assert e2.stats()["suspended"] == 1
        sid, off = e2.stream_resume_saved(want, 0)                     # the size comes from the saved record
        assert off == saved
        _write(e2, sid, body, start=saved)                             # upstream answers Range: bytes=<saved>-
        dig, ok = e2.stream_finish(sid)
        assert ok and dig == want
        assert e2.fetch(want, chunk=4 << 20) == body.tobytes()
        assert e2.stats()["suspended"] == 0 and os.listdir(os.path.join(cas, "partial")) == []
        if resume_on == "disk":
            _check_published(e2, cas, body, dig)


def test_disk_only_engine_caches_every_body_on_disk(tmp_path):
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    with _engine(cas, flags=DM_F_NO_HBM_CAS | DM_F_DISK_DIRECT) as eng:
        used0 = eng.stats()["hbm_cas_used"]
        for seed, n in ((8, 0), (9, 1000), (10, 65), (11, ARENA + ARENA // 2 + 3)):
            body = _body(seed, n)
            dig, ok = eng.ingest(body, expect=hashlib.sha256(body.tobytes()).digest(), chunk=1 << 20)
            assert ok
            _check_published(eng, cas, body, dig)
        assert eng.stats()["hbm_cas_used"] == used0


def test_disk_sync_file_exists_when_finish_returns(tmp_path):
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_DISK_SYNC
    cas = str(tmp_path / "cas")
    body = _body(12, ARENA + ARENA // 2 + 5)
    with _engine(cas, flags=DM_F_DISK_DIRECT | DM_F_DISK_SYNC) as eng:
        dig, ok = eng.ingest(body, chunk=1 << 20)
        assert ok and os.path.getsize(_blob_file(cas, dig)) == body.nbytes


def test_four_gib_body(tmp_path):
    """One body of 4 GiB + 65 bytes: offsets past 2^32 in the file, the job chain and the sidecar."""
    n = (4 << 30) + 65
    if shutil.disk_usage(str(tmp_path)).free < 3 * n:
        pytest.skip("needs three times the body size free on the temporary filesystem")
    cas = str(tmp_path / "cas")
    h = hashlib.sha256()
    piece = _body(13, 64 << 20)
    with _engine(cas) as eng:
        sid = eng.stream_open(None, n)
        left, k = n, 0
        while left:
            m = min(left, piece.nbytes)
            chunk = piece[:m] if k % 2 == 0 else piece[::-1][:m].copy()
            h.update(chunk.tobytes())
            eng.stream_write(sid, chunk)
            left -= m
            k += 1
        eng.stream_flush(sid)
        dig, ok = eng.stream_finish(sid)
        assert ok and dig == h.digest()
        path = _blob_file(cas, dig)
        assert os.path.getsize(path) == n
        hf = hashlib.sha256()
        with open(path, "rb") as f:
            for b in iter(lambda: f.read(64 << 20), b""):
                hf.update(b)
        assert hf.digest() == dig
