"""dm_cache_remove, dm_cache_alias_del and dm_cache_alias_list on the GPU: removal from both tiers, what readers that
already had a blob open keep, refusals while a digest is being placed or loaded, alias tombstones that survive a restart,
listing pages, and tools/dm_rm.py over imported HuggingFace and Ollama layouts.

Sizes are module constants so that tests/test_remove_host.py can run the same tests over the fake CUDA runtime with a
small arena."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARENA = 256 << 20           # HBM arena of the engines
RING = 64 << 20
BIG = 64 << 20              # blobs whose spill or load is still running when the removal comes
MID = 8 << 20               # the blob readers have open during a removal
PIECE = 32 << 10


def _d2h(ptr, n):
    """Bytes [ptr, ptr + n) of device memory."""
    import torch

    class _Dev:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy().tobytes()


def _to_dev(host):
    """(device pointer, owner) of a device copy of a uint8 array."""
    import torch
    t = torch.from_numpy(host).cuda()
    return t.data_ptr(), t


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes()).digest()


def _engine(cas=None, hbm=None, **kw):
    import demodel_b200
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, ring_bytes=RING, cas_dir=cas, **kw)


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for off in range(0, body.nbytes, 4 << 20):
        eng.stream_write(sid, body[off:off + (4 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _read_all(eng, rid, size, start=0, piece=PIECE):
    got = bytearray()
    while start + len(got) < size:
        part = eng.cache_read(rid, start + len(got), min(piece, size - start - len(got)))
        assert part
        got += part
    return bytes(got)


def _names_for(cas, dig):
    d = os.path.join(cas, "blobs", "sha256", dig.hex()[:2])
    return sorted(n for n in os.listdir(d) if n.startswith(dig.hex())) if os.path.isdir(d) else []


def _walk(cas):
    total = 0
    for sub in ("blobs", "incoming", "partial"):
        for dirpath, _, files in os.walk(os.path.join(cas, sub)):
            total += sum(os.path.getsize(os.path.join(dirpath, f)) for f in files)
    return total


def _clean(eng, max_streams=65536, readers=0):
    for _ in range(1000):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == readers):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def test_hbm_only_removal_frees_the_extent(tmp_path):
    import demodel_b200
    with _engine() as eng:
        bodies = [_body(1, MID), _body(2, 4096)]
        digs = [_ingest(eng, b) for b in bodies]
        used = eng.stats()["hbm_cas_used"]
        assert eng.cache_remove([digs[0]]) == [demodel_b200.DM_OK]
        assert eng.cache_contains(digs[0]) is None and eng.cache_open(digs[0]) is None
        assert eng.cache_open_verified(digs[0]) is None and eng.promote([digs[0]]) == [demodel_b200.DM_ENOENT]
        assert eng.stats()["hbm_cas_used"] == used - MID
        assert eng.fetch(digs[1]) == bodies[1].tobytes()                 # the other blob is untouched
        assert eng.cache_remove([digs[0]], partial=True) == [demodel_b200.DM_ENOENT]
        other = _body(3, MID)                                             # the freed space is reused
        _ingest(eng, other)
        assert eng.stats()["hbm_cas_used"] == used
        _clean(eng)


def test_both_tiers_and_restart(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    bodies = [_body(10 + i, 100_000 + i) for i in range(3)]
    with _engine(cas, flags=demodel_b200._lib.DM_F_DISK_SYNC) as eng:
        digs = [_ingest(eng, b) for b in bodies]
        for d in digs:
            assert _names_for(cas, d) == [d.hex(), d.hex() + ".meta"]
        committed = eng.stats()["blobs_committed"]
        assert eng.cache_remove([digs[1], digs[1]]) == [demodel_b200.DM_OK] * 2      # a duplicate is handled once
        assert _names_for(cas, digs[1]) == []
        assert [d for d, _ in eng.list()] == sorted([digs[0], digs[2]])
        assert eng.cache_contains(digs[1]) is None and eng.cache_follow(digs[1]) is None
        assert eng.stats()["blobs_committed"] == committed
        _clean(eng)
    with _engine(cas) as eng:
        assert eng.cache_open(digs[1]) is None and eng.cache_contains(digs[1]) is None
        assert eng.fetch(digs[0]) == bodies[0].tobytes()
        assert eng.cache_remove([digs[0]]) == [demodel_b200.DM_OK]                  # disk only
        assert eng.cache_open(digs[0]) is None and _names_for(cas, digs[0]) == []


def test_hbm_reader_keeps_its_extent(tmp_path):
    import demodel_b200
    with _engine() as eng:
        body = _body(20, MID)
        dig = _ingest(eng, body)
        used = eng.stats()["hbm_cas_used"]
        rid, size = eng.cache_open(dig)
        first = _read_all(eng, rid, size // 2)
        assert eng.cache_remove([dig]) == [demodel_b200.DM_OK]
        assert eng.cache_open(dig) is None and eng.cache_contains(dig) is None
        assert eng.cache_evict(dig) is False
        assert eng.stats()["hbm_cas_used"] == used                         # still read
        rest = _read_all(eng, rid, size, start=size // 2)
        assert first + rest == body.tobytes()
        ext = eng.cache_device_extents(rid)
        assert b"".join(_d2h(p, n) for p, n in ext if n) == body.tobytes()
        eng.cache_close(rid)
        assert eng.stats()["hbm_cas_used"] == used - MID
        _clean(eng)


def test_disk_reader_reads_to_eof(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(30, MID)
    with _engine(cas, flags=demodel_b200._lib.DM_F_DISK_SYNC) as eng:
        dig = _ingest(eng, body)
    with _engine(cas) as eng:
        rid, size = eng.cache_open(dig)                                   # disk tier only
        assert eng.cache_remove([dig]) == [demodel_b200.DM_OK]
        assert _names_for(cas, dig) == [] and eng.cache_open(dig) is None
        assert _read_all(eng, rid, size) == body.tobytes()
        assert eng.cache_read(rid, size, PIECE) == b""
        eng.cache_close(rid)
        _clean(eng)


def test_removal_during_a_running_spill(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(40, BIG)
    with _engine(cas) as eng:                                             # no DM_F_DISK_SYNC: finish does not wait
        dig = _ingest(eng, body)
        assert eng.cache_remove([dig]) == [demodel_b200.DM_OK]
    assert _names_for(cas, dig) == []                                     # no file, no .part, no sidecar


def test_refused_while_placed_or_loaded(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    bodies = [_body(50, BIG), _body(51, BIG), _body(52, 5000)]
    with _engine(cas, flags=demodel_b200._lib.DM_F_DISK_SYNC) as eng:
        digs = [_ingest(eng, b) for b in bodies]
    with _engine(cas) as eng:
        # a stream that expects the digest
        sid = eng.stream_open(digs[2], 5000)
        assert eng.cache_remove([digs[2]]) == [demodel_b200.DM_ESTATE]
        assert digs[2].hex() in eng.error_detail(0) and "stream" in eng.error_detail(0)
        assert eng.fetch(digs[2]) == bodies[2].tobytes()                  # nothing of it was removed
        eng.stream_abort(sid)
        # a running verified-open load
        rid, size = eng.cache_open_verified(digs[0])
        assert eng.cache_remove([digs[0]]) == [demodel_b200.DM_ESTATE]
        assert "load" in eng.error_detail(0)
        assert _read_all(eng, rid, size) == bodies[0].tobytes()
        eng.cache_close(rid)
        # a running promotion
        out = {}
        th = threading.Thread(target=lambda: out.setdefault("st", eng.promote([digs[1]])))
        slots = eng.stats()["free_stream_slots"]
        th.start()
        while th.is_alive() and eng.stats()["free_stream_slots"] == slots:   # until the load's stream is open
            pass
        refused = eng.cache_remove([digs[1]]) if th.is_alive() else [demodel_b200.DM_ESTATE]   # (or it was quicker)
        th.join()
        assert refused == [demodel_b200.DM_ESTATE] and out["st"] == [demodel_b200.DM_OK], (refused, out)
        assert eng.cache_remove(digs) == [demodel_b200.DM_OK] * 3         # each has ended
        assert all(_names_for(cas, d) == [] for d in digs)
        _clean(eng)


def test_aliases_tombstones_and_restart(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    bodies = [_body(60 + i, 3000 + i) for i in range(3)]
    with _engine(cas) as eng:
        digs = [_ingest(eng, b) for b in bodies]
        eng.alias_put("https://h/a/resolve/main/x", digs[0])
        eng.alias_put("https://h/b/resolve/main/x", digs[1])
        eng.alias_put("https://h/b/resolve/main/y", digs[1])
        eng.alias_put("https://h/c/resolve/main/z", digs[2])
        assert eng.cache_remove([digs[0]]) == [demodel_b200.DM_OK]        # without DM_RM_ALIASES: they stay
        assert eng.alias_get("https://h/a/resolve/main/x") == digs[0]
        assert eng.proxy_request("https://h/a/resolve/main/x") is None
        assert eng.cache_remove([digs[1], digs[0]], aliases=True) == [demodel_b200.DM_OK, demodel_b200.DM_ENOENT]
        assert eng.alias_get("https://h/b/resolve/main/x") is None and eng.alias_get("https://h/a/resolve/main/x") is None
        assert eng.alias_del("https://h/c/resolve/main/z") and not eng.alias_del("https://h/c/resolve/main/z")
        assert eng.stats()["aliases"] == 0
        eng.alias_put("https://h/c/resolve/main/z", digs[2])              # put after a deletion wins at replay
        assert eng.stats()["blobs_committed"] == 3
    with open(os.path.join(cas, "aliases.log")) as f:
        assert sum(line.startswith("-\t") for line in f) == 4
    with _engine(cas) as eng:
        assert eng.alias_get("https://h/b/resolve/main/y") is None and eng.alias_get("https://h/a/resolve/main/x") is None
        assert eng.alias_get("https://h/c/resolve/main/z") == digs[2]
        assert list(eng.alias_list()) == [("https://h/c/resolve/main/z", digs[2])]


def test_alias_log_compacted_after_many_deletions(tmp_path):
    cas = str(tmp_path / "cas")
    dig = hashlib.sha256(b"x").digest()
    with _engine(cas) as eng:
        for i in range(3000):
            eng.alias_put(f"k{i:05d}", dig)
        for i in range(2990):
            assert eng.alias_del(f"k{i:05d}")
    log = os.path.join(cas, "aliases.log")
    with open(log) as f:
        assert len(f.readlines()) == 5990
    with _engine(cas) as eng:                                             # replayed, then rewritten
        assert [k for k, _ in eng.alias_list()] == [f"k{i:05d}" for i in range(2990, 3000)]
    with open(log) as f:
        lines = f.readlines()
    assert len(lines) == 10 and not any(line.startswith("-") for line in lines)
    with _engine(cas) as eng:
        assert eng.stats()["aliases"] == 10


def test_alias_list_pages(tmp_path):
    import demodel_b200
    keys = ["a", "ab", "abc", "b", "b/été", "b/日本", "b/z", "c" * 4096, "é"]
    with _engine() as eng:
        for i, k in enumerate(keys):
            eng.alias_put(k, bytes([i]) * 32)
        want = sorted(keys, key=lambda k: k.encode())
        assert [k for k, _ in eng.alias_list()] == want
        assert [k for k, _ in eng.alias_list(page=1, keys_bytes=4097)] == want
        assert [(k, d) for k, d in eng.alias_list("b/")] == [(k, bytes([keys.index(k)]) * 32) for k in want if k.startswith("b/")]
        assert [k for k, _ in eng.alias_list("é")] == ["é"]
        lib, h = eng._lib, eng._h
        buf = C.create_string_buffer(16)
        digs = (C.c_uint8 * (32 * 8))()
        n, more = C.c_uint32(), C.c_int()
        assert lib.dm_cache_alias_list(h, b"a", None, buf, 16, digs, 8, C.byref(n), C.byref(more)) == 0
        assert (n.value, more.value) == (3, 0) and buf.raw[:9] == b"a\0ab\0abc\0"
        assert lib.dm_cache_alias_list(h, b"", b"ab", buf, 16, digs, 8, C.byref(n), C.byref(more)) == 0
        assert (n.value, more.value) == (3, 1)                             # the next key does not fit
        assert buf.raw[:10] == b"abc\0b\0b/z\0"                         # (é is 0xc3 0xa9: after z)
        assert lib.dm_cache_alias_list(h, b"", b"b", buf, 16, digs, 1, C.byref(n), C.byref(more)) == 0
        assert (n.value, more.value) == (1, 1) and bytes(digs[:32]) == bytes([6]) * 32       # cap reached: b/z
        assert lib.dm_cache_alias_list(h, b"b", b"a", buf, 16, digs, 8, C.byref(n), C.byref(more)) == 0
        assert n.value >= 1 and buf.raw[:2] == b"b\0"                      # an `after` below the prefix skips nothing
        assert lib.dm_cache_alias_list(h, b"zz", None, None, 0, None, 0, C.byref(n), C.byref(more)) == 0
        assert (n.value, more.value) == (0, 0)
        assert lib.dm_cache_alias_list(h, b"", None, None, 0, None, 0, C.byref(n), C.byref(more)) == 0
        assert (n.value, more.value) == (0, 1)
        assert lib.dm_cache_alias_list(h, b"", None, None, 16, digs, 8, C.byref(n), C.byref(more)) == demodel_b200.DM_EINVAL


def test_partial_removes_a_saved_download(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(70, 3 << 20)
    dig = _sha(body)
    with _engine(cas) as eng:
        sid = eng.stream_open(dig, body.nbytes)
        eng.stream_write(sid, body[:1 << 20])
        assert eng.stream_suspend(sid) > 0
        assert eng.stats()["suspended"] == 1
        assert eng.cache_remove([dig]) == [demodel_b200.DM_ENOENT]          # without DM_RM_PARTIAL it stays
        assert eng.cache_remove([dig], partial=True) == [demodel_b200.DM_OK]
        assert eng.stats()["suspended"] == 0 and os.listdir(os.path.join(cas, "partial")) == []
        assert eng.stream_resume_saved(dig, body.nbytes) is None
        _clean(eng)


def test_limit_index_matches_the_directories(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    bodies = [_body(80 + i, 200_000 + 1000 * i) for i in range(6)]
    with _engine(cas, flags=demodel_b200._lib.DM_F_DISK_SYNC) as eng:
        digs = [_ingest(eng, b) for b in bodies]
        sid = eng.stream_open(_sha(_body(99, 1 << 20)), 1 << 20)
        eng.stream_write(sid, _body(99, 1 << 20)[:1 << 19])
        eng.stream_suspend(sid)
        eng.set_disk_limit(1 << 40)
        before = eng.disk_usage()
        assert before["used_bytes"] == _walk(cas)
        assert eng.cache_remove(digs[:3] + [_sha(_body(99, 1 << 20))], partial=True) == [demodel_b200.DM_OK] * 4
        after = eng.disk_usage()
        assert after["used_bytes"] == _walk(cas) and after["blob_files"] == 3 and after["partial_bytes"] == 0
        for k in ("evicted_files", "evicted_bytes", "refused"):
            assert after[k] == before[k]
        _clean(eng)


def test_removal_races_a_replacing_ingest(tmp_path):
    import demodel_b200
    n, size = 64, 8192
    host = _body(90, n * size)
    offs, lens = [i * size for i in range(n)], [size] * n
    exp = b"".join(_sha(host[o:o + size]) for o in offs)
    digs = [exp[32 * i:32 * i + 32] for i in range(n)]
    dev, keep = _to_dev(host)
    with _engine() as eng:
        eng.ingest_device(dev, offs, lens, expect=exp)
        seen = set()
        stop = threading.Event()

        def reingest():
            while not stop.is_set():
                eng.ingest_device(dev, offs, lens, expect=exp, replace=True)
        th = threading.Thread(target=reingest)
        th.start()
        try:
            for _ in range(20):
                st = eng.cache_remove(digs)
                assert set(st) <= {demodel_b200.DM_OK, demodel_b200.DM_ENOENT, demodel_b200.DM_ESTATE}
                seen |= set(st)
        finally:
            stop.set()
            th.join()
        for d, o in zip(digs, offs):                                      # consistent: a hit serves the blob, or a miss
            got = eng.fetch(d)
            assert got is None or got == host[o:o + size].tobytes()
        assert set(eng.cache_remove(digs)) <= {demodel_b200.DM_OK, demodel_b200.DM_ENOENT}
        assert all(eng.cache_contains(d) is None for d in digs)
        assert eng.stats()["hbm_cas_used"] == 0
        eng.ingest_device(dev, offs, lens, expect=exp)                    # not a ban
        assert all(eng.fetch(d) == host[o:o + size].tobytes() for d, o in zip(digs, offs))
        _clean(eng)
    del keep


def test_reingest_after_removal(tmp_path):
    import demodel_b200
    cas = str(tmp_path / "cas")
    body = _body(100, 300_000)
    with _engine(cas, flags=demodel_b200._lib.DM_F_DISK_SYNC) as eng:
        dig = _ingest(eng, body)
        assert eng.cache_remove([dig], aliases=True, partial=True) == [demodel_b200.DM_OK]
        assert _ingest(eng, body) == dig
        assert eng.fetch(dig) == body.tobytes() and _names_for(cas, dig) == [dig.hex(), dig.hex() + ".meta"]
        assert eng.stats()["blobs_committed"] == 2


def test_arguments(tmp_path):
    import demodel_b200
    lib = demodel_b200.load()
    with _engine() as eng:
        st = (C.c_int32 * 2)()
        assert lib.dm_cache_remove(eng._h, None, 0, 0, None) == 0
        assert lib.dm_cache_remove(eng._h, None, 1, 0, st) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_remove(eng._h, bytes(32), 1, 0, None) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_remove(eng._h, bytes(32), 1, 0x4, st) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_remove(None, bytes(32), 1, 0, st) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_remove(eng._h, bytes(32), 1, 3, st) == 0 and st[0] == demodel_b200.DM_ENOENT
        assert lib.dm_cache_alias_del(eng._h, None) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_alias_del(eng._h, b"nope") == demodel_b200.DM_ENOENT
        n, more = C.c_uint32(), C.c_int()
        assert lib.dm_cache_alias_list(eng._h, None, None, None, 0, None, 0, None, C.byref(more)) == demodel_b200.DM_EINVAL
        assert lib.dm_cache_alias_list(eng._h, None, None, None, 0, None, 0, C.byref(n), C.byref(more)) == 0
        assert eng.cache_remove([]) == []


def _dm_rm(cas, *args):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dm_rm.py"), "--cas-dir", cas, *args],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_dm_rm_hf_repositories_sharing_a_file(tmp_path):
    from demodel_b200 import importer
    hub = tmp_path / "hub"
    shared = b'{"tokenizer": 1}' * 100
    files = {"org--a": {"tokenizer.json": shared, "model.bin": b"A" * 70000},
             "org--b": {"tokenizer.json": shared, "model.bin": b"B" * 70000}}
    for repo, content in files.items():
        base = hub / f"models--{repo}"
        (base / "refs").mkdir(parents=True)
        (base / "refs" / "main").write_text("c" * 40)
        (base / "blobs").mkdir()
        snap = base / "snapshots" / ("c" * 40)
        snap.mkdir(parents=True)
        for name, data in content.items():
            h = hashlib.sha256(data).hexdigest()
            (base / "blobs" / h).write_bytes(data)
            os.symlink(base / "blobs" / h, snap / name)
    cas = str(tmp_path / "cas")
    with _engine(cas) as eng:
        importer.import_entries(eng, importer.hf_entries(str(hub)))
    plan = _dm_rm(cas, "--hf-repo", "org/a", "--dry-run")
    assert plan["removed"] == [hashlib.sha256(b"A" * 70000).hexdigest()] and plan["bytes_freed"] == 70000
    assert plan["kept"] == [hashlib.sha256(shared).hexdigest()]
    with _engine(cas) as eng:
        assert len(eng.list()) == 3                                       # a dry run removes nothing
    res = _dm_rm(cas, "--hf-repo", "org/a")
    assert res["removed"] == plan["removed"] and res["bytes_freed"] == 70000
    with _engine(cas) as eng:
        left = {d.hex() for d, _ in eng.list()}
        assert left == {hashlib.sha256(shared).hexdigest(), hashlib.sha256(b"B" * 70000).hexdigest()}
        assert list(eng.alias_list(importer.HF_ENDPOINT + "/org/a/")) == []
        assert len(list(eng.alias_list(importer.HF_ENDPOINT + "/org/b/"))) == 4


def test_dm_rm_ollama_models_sharing_a_layer(tmp_path):
    from demodel_b200 import importer
    models = tmp_path / "models"
    (models / "blobs").mkdir(parents=True)
    licence, w1, w2 = b"MIT licence" * 50, b"W" * 90000, b"V" * 90000

    def blob(data):
        h = hashlib.sha256(data).hexdigest()
        (models / "blobs" / f"sha256-{h}").write_bytes(data)
        return h

    for model, weights in (("one", w1), ("two", w2)):
        cfg = json.dumps({"model": model}).encode()
        layers = [(licence, "application/vnd.ollama.image.license"), (weights, "application/vnd.ollama.image.model")]
        man = json.dumps({"schemaVersion": 2, "mediaType": "application/vnd.docker.distribution.manifest.v2+json",
                          "config": {"mediaType": "application/vnd.docker.container.image.v1+json",
                                     "digest": "sha256:" + blob(cfg), "size": len(cfg)},
                          "layers": [{"mediaType": m, "digest": "sha256:" + blob(d), "size": len(d)} for d, m in layers]})
        d = models / "manifests" / "registry.ollama.ai" / "library" / model
        d.mkdir(parents=True)
        (d / "latest").write_text(man)
    cas = str(tmp_path / "cas")
    with _engine(cas) as eng:
        importer.import_entries(eng, importer.ollama_entries(str(models)))
        before = {d.hex() for d, _ in eng.list()}
    assert len(before) == 7                                               # 2 configs, licence, 2 weights, 2 manifests
    res = _dm_rm(cas, "--ollama", "https://registry.ollama.ai/v2/library/one/manifests/latest")
    assert len(res["removed"]) == 3 and hashlib.sha256(w1).hexdigest() in res["removed"]
    assert res["kept"] == [hashlib.sha256(licence).hexdigest()]
    with _engine(cas) as eng:
        left = {d.hex() for d, _ in eng.list()}
        assert left == before - set(res["removed"]) and hashlib.sha256(licence).hexdigest() in left
        assert eng.alias_get("https://registry.ollama.ai/v2/library/one/manifests/latest") is None
        assert eng.alias_get("https://registry.ollama.ai/v2/library/two/manifests/latest") is not None


def test_nothing_leaks(tmp_path):
    """Slabs, stream slots and readers are all back after removals with readers, a spill and refusals."""
    import demodel_b200
    cas = str(tmp_path / "cas")
    with _engine(cas, max_streams=256) as eng:
        bodies = [_body(110 + i, 50_000 * (i + 1)) for i in range(4)]
        digs = [_ingest(eng, b) for b in bodies]
        rids = [eng.cache_open(d)[0] for d in digs[:2]]
        sid = eng.stream_open(digs[3], bodies[3].nbytes)
        assert eng.cache_remove(digs, partial=True) == [demodel_b200.DM_OK] * 3 + [demodel_b200.DM_ESTATE]
        for r in rids:
            eng.cache_close(r)
        eng.stream_abort(sid)
        assert eng.cache_remove(digs) == [demodel_b200.DM_ENOENT] * 3 + [demodel_b200.DM_OK]
        _clean(eng, max_streams=256)
        assert eng.stats()["hbm_cas_used"] == 0
