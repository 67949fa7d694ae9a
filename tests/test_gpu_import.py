"""dm_cache_import on the GPU: files from outside the cache are staged under <cas_dir>/incoming/, hashed there by the
SHA-256 kernels (read back through the ring by the disk threads, or through packs at most tiny_max bytes) and renamed
into the disk tier, without touching the HBM arena.  Every digest is checked against hashlib over the source bytes.

Sizes are module constants so that tests/test_import_host.py can run the same tests over the fake CUDA runtime with a
small ring and arena."""
import contextlib
import hashlib
import io
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARENA = 512 << 20           # HBM arena of the importing engines
RING = 64 << 20
SLAB = 1 << 20
SMALL_ARENA = 16 << 20      # the arena a file larger than it is imported next to
BIG = 96 << 20              # the largest of the sizes that matter
HUGE = (4 << 30) + 65       # crosses 2^32 by a block and a byte
MANY = 3000                 # tiny files (at most 8 KiB) in one call
LIVE_FILES = 64             # multi-slab files imported while live writers stream


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


def _write(path, body):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(body.tobytes() if isinstance(body, np.ndarray) else body)
    return path


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for off in range(0, body.nbytes, 1 << 20):
        eng.stream_write(sid, body[off:off + (1 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _incoming(cas):
    d = os.path.join(cas, "incoming")
    return sorted(os.listdir(d)) if os.path.isdir(d) else []


def _file_hash(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 24), b""):
            h.update(chunk)
    return h.digest()


def _tree_state(root):
    """Every file and link under root: content hash (or link target), inode and mtime."""
    out = {}
    for dirpath, _, files in os.walk(root):
        for f in files:
            p = os.path.join(dirpath, f)
            st = os.lstat(p)
            what = os.readlink(p) if os.path.islink(p) else _file_hash(p)
            out[os.path.relpath(p, root)] = (what, st.st_ino, st.st_mtime_ns)
    return out


def _clean(eng, max_streams=65536):
    import time
    for _ in range(400):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == 0):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _sidecar_size(cas, dig):
    with open(_blob_file(cas, dig) + ".meta") as f:
        meta = json.load(f)
    assert meta["digest"] == "sha256:" + dig.hex() and meta["encoding"] == "identity" and meta["headers"] == {}
    return meta["size"]


def test_sizes_that_matter_with_known_and_unknown_digests(tmp_path):
    from demodel_b200 import DM_OK
    cas, src = str(tmp_path / "cas"), tmp_path / "src"
    sizes = [0, 1, 55, 56, 63, 64, 65, 64 << 10, (64 << 10) + 1, (1 << 20) + 7, BIG]
    bodies = [_body(100 + i, n) for i, n in enumerate(sizes)]
    paths = [_write(str(src / f"f{i}"), b) for i, b in enumerate(bodies)]
    digs = [_sha(b) for b in bodies]
    half = len(sizes) // 2
    expect = [d if i < half else None for i, d in enumerate(digs)]          # the first half by name, the rest unknown
    with _engine(cas) as eng:
        st0 = eng.stats()
        res = eng.import_files(paths, expect=expect)
        st = eng.stats()
        assert res == [(DM_OK, d) for d in digs]
        assert st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert st["bytes_hashed"] - st0["bytes_hashed"] == sum(sizes)
        assert st["h2d_bytes"] - st0["h2d_bytes"] == sum(sizes)
        assert st["blobs_committed"] - st0["blobs_committed"] == len(sizes)
        assert st["bytes_ingested"] == st0["bytes_ingested"] and st["blobs_mismatched"] == st0["blobs_mismatched"]
        for d, b, p in zip(digs, bodies, paths):
            assert _file_hash(_blob_file(cas, d)) == d and os.path.getsize(_blob_file(cas, d)) == b.nbytes
            assert _sidecar_size(cas, d) == b.nbytes
            assert os.stat(_blob_file(cas, d)).st_ino != os.stat(p).st_ino                # a copy, not a link
            assert eng.fetch(d, chunk=4 << 20) == b.tobytes()
        assert sorted(eng.list()) == sorted((d, b.nbytes) for d, b in zip(digs, bodies))
        assert eng.verify(digs) == [DM_OK] * len(digs)
        assert _incoming(cas) == []
        _clean(eng)
    with _engine(cas) as eng:                                                # a fresh engine serves every blob
        for d, b in zip(digs, bodies):
            assert eng.fetch(d, chunk=4 << 20) == b.tobytes()
        assert eng.promote(digs) == [DM_OK] * len(digs)
        _clean(eng)
    for p, b in zip(paths, bodies):
        assert _file_hash(p) == _sha(b)


@pytest.mark.parametrize("mode", ["small_arena", "no_hbm", "disk_direct"])
def test_file_larger_than_the_arena_in_every_engine_mode(tmp_path, mode):
    from demodel_b200 import DM_OK
    from demodel_b200._lib import DM_F_DISK_DIRECT, DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    body = _body(300, SMALL_ARENA + 12345)
    p = _write(str(tmp_path / "src" / "big"), body)
    flags = {"small_arena": 0, "no_hbm": DM_F_NO_HBM_CAS, "disk_direct": DM_F_DISK_DIRECT}[mode]
    with _engine(cas, hbm=SMALL_ARENA, flags=flags) as eng:
        used = eng.stats()["hbm_cas_used"]
        assert eng.import_files([p], expect=[None]) == [(DM_OK, _sha(body))]
        assert eng.stats()["hbm_cas_used"] == used
        assert eng.fetch(_sha(body), chunk=4 << 20) == body.tobytes()
        assert eng.verify([_sha(body)]) == [DM_OK]
        assert _incoming(cas) == []
        _clean(eng)


def test_a_file_beyond_4_gib(tmp_path):
    from demodel_b200 import DM_OK
    from demodel_b200.engine import synth_fill_host
    cas = str(tmp_path / "cas")
    p = str(tmp_path / "huge.safetensors")
    h = hashlib.sha256()
    step = 1 << 30
    with open(p, "wb") as f:                                                 # generated on the host, as test_gpu_large.py does
        for lo in range(0, HUGE, step):
            part = synth_fill_host(0xDE40DE1, 9200, lo, min(step, HUGE - lo))
            h.update(part)
            f.write(part.tobytes())
    want = h.digest()
    with _engine(cas, hbm=SMALL_ARENA) as eng:
        st0 = eng.stats()
        assert eng.import_files([p], expect=[want], link=True) == [(DM_OK, want)]
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == HUGE and st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert os.path.getsize(_blob_file(cas, want)) == HUGE and _sidecar_size(cas, want) == HUGE
        rid, size = eng.cache_open(want)
        assert size == HUGE
        lo = min(4 << 30, HUGE) - 64
        assert eng.cache_read(rid, lo, 129) == synth_fill_host(0xDE40DE1, 9200, lo, min(129, HUGE - lo)).tobytes()
        eng.cache_close(rid)
        assert _incoming(cas) == []
        _clean(eng)


def test_wrong_inputs(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_ECORRUPT, DM_EINVAL, DM_ENOENT, DM_ESTATE
    cas = str(tmp_path / "cas")
    n = 3 * SLAB + 100
    bodies = [_body(400, n), _body(401, n), _body(402, n), _body(403, 5000)]
    paths = [_write(str(tmp_path / "src" / f"f{i}"), b) for i, b in enumerate(bodies)]
    wrong = []
    for b, at in zip(bodies, (0, 15, 31, 16)):                              # one flipped byte at the start, middle, end
        d = bytearray(_sha(b))
        d[at] ^= 0x01
        wrong.append(bytes(d))
    before = _tree_state(str(tmp_path / "src"))
    with _engine(cas) as eng:
        st0 = eng.stats()
        res = eng.import_files(paths + [str(tmp_path / "missing"), str(tmp_path / "src")], expect=wrong + [None, None])
        assert res[:4] == [(DM_ECORRUPT, _sha(b)) for b in bodies]           # the real digest comes back
        assert res[4] == (DM_ENOENT, bytes(32)) and res[5] == (DM_EINVAL, bytes(32))
        st = eng.stats()
        assert st["blobs_committed"] == st0["blobs_committed"] and st["blobs_mismatched"] == st0["blobs_mismatched"]
        assert eng.list() == [] and _incoming(cas) == []
        for b in bodies:
            assert eng.cache_contains(_sha(b)) is None
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.import_files([paths[0]], keys=["bad\nkey"])
        assert ei.value.code == DM_EINVAL
        _clean(eng)
    assert _tree_state(str(tmp_path / "src")) == before
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, slab_bytes=SLAB) as eng:
        with pytest.raises(demodel_b200.DmError) as ei:
            eng.import_files(paths)
        assert ei.value.code == DM_ESTATE


def test_already_cached_and_duplicates(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    cached, fresh = _body(500, 2 * SLAB + 5), _body(501, 3 * SLAB + 9)
    with _engine(cas) as eng:
        _ingest(eng, cached)
    ino = os.stat(_blob_file(cas, _sha(cached))).st_ino
    pc = _write(str(tmp_path / "src" / "cached"), cached)
    pf = _write(str(tmp_path / "src" / "fresh"), fresh)
    with _engine(cas) as eng:
        st0 = eng.stats()
        res = eng.import_files([pc, pf, pf, pf], expect=[_sha(cached), None, None, None],
                               keys=["https://h/cached", "https://h/a", None, "https://h/b"])
        st = eng.stats()
        assert res == [(DM_OK, _sha(cached))] + [(DM_OK, _sha(fresh))] * 3
        assert st["bytes_hashed"] - st0["bytes_hashed"] == fresh.nbytes          # the cached one is not read, the
        assert st["blobs_committed"] - st0["blobs_committed"] == 1              # duplicate is hashed once
        assert os.stat(_blob_file(cas, _sha(cached))).st_ino == ino
        assert eng.alias_get("https://h/cached") == _sha(cached)
        assert eng.alias_get("https://h/a") == eng.alias_get("https://h/b") == _sha(fresh)
        # an unknown digest that turns out to be cached: hashed, and the tier's copy stays
        st0 = eng.stats()
        assert eng.import_files([pc]) == [(DM_OK, _sha(cached))]
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == cached.nbytes and st["blobs_committed"] == st0["blobs_committed"]
        assert os.stat(_blob_file(cas, _sha(cached))).st_ino == ino and _incoming(cas) == []
        _clean(eng)


def test_links(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    body, small = _body(600, 2 * SLAB + 1), _body(601, 3000)
    blob = _write(str(tmp_path / "hub" / "blobs" / _sha(body).hex()), body)
    snap = tmp_path / "hub" / "snapshots" / "abc"
    snap.mkdir(parents=True)
    os.symlink(os.path.join("..", "..", "blobs", _sha(body).hex()), snap / "model.bin")
    ps = _write(str(tmp_path / "small"), small)
    with _engine(cas) as eng:
        res = eng.import_files([str(snap / "model.bin"), ps], expect=[_sha(body), None], link=True)
        assert res == [(DM_OK, _sha(body)), (DM_OK, _sha(small))]
        assert os.stat(_blob_file(cas, _sha(body))).st_ino == os.stat(blob).st_ino     # the link goes to the target
        assert os.stat(_blob_file(cas, _sha(small))).st_ino == os.stat(ps).st_ino
        assert os.path.islink(snap / "model.bin") and _file_hash(blob) == _sha(body)
        assert eng.fetch(_sha(body), chunk=4 << 20) == body.tobytes()
        assert _incoming(cas) == []
        _clean(eng)


def test_link_across_filesystems_falls_back_to_a_copy(tmp_path):
    import tempfile
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    shm = "/dev/shm"
    os.makedirs(cas)
    if not (os.path.isdir(shm) and os.access(shm, os.W_OK) and os.stat(shm).st_dev != os.stat(cas).st_dev):
        pytest.skip("no second filesystem (/dev/shm) to check the EXDEV fall-back on")
    other = _body(602, SLAB + 3)
    with tempfile.TemporaryDirectory(dir=shm) as d, _engine(cas) as eng:
        po = _write(os.path.join(d, "other"), other)
        assert eng.import_files([po], link=True) == [(DM_OK, _sha(other))]
        assert os.stat(_blob_file(cas, _sha(other))).st_ino != os.stat(po).st_ino
        assert _file_hash(_blob_file(cas, _sha(other))) == _sha(other) and _file_hash(po) == _sha(other)
        assert _incoming(cas) == []
        _clean(eng)


def test_many_small_files_share_launches(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    rng = np.random.default_rng(700)
    sizes = rng.integers(1, 8192, MANY)
    src = tmp_path / "src"
    src.mkdir()
    paths, digs = [], []
    for i, n in enumerate(sizes):
        b = rng.integers(0, 256, int(n), dtype=np.uint8)
        paths.append(_write(str(src / f"{i:05d}"), b))
        digs.append(_sha(b))
    with _engine(cas) as eng:
        st0 = eng.stats()
        res = eng.import_files(paths, expect=[d if i % 2 else None for i, d in enumerate(digs)])
        st = eng.stats()
        assert res == [(DM_OK, d) for d in digs]
        assert st["kernel_launches"] - st0["kernel_launches"] < 300              # the chains went out together
        assert st["bytes_hashed"] - st0["bytes_hashed"] == int(sizes.sum())
        assert st["h2d_bytes"] - st0["h2d_bytes"] == int(sizes.sum())
        assert st["hbm_cas_used"] == st0["hbm_cas_used"]
        assert _incoming(cas) == []
        _clean(eng)


def test_import_races_a_stream_and_a_verify(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(800 + i, (i + 1) * 300001) for i in range(6)]
    paths = [_write(str(tmp_path / "src" / f"f{i}"), b) for i, b in enumerate(bodies)]
    digs = [_sha(b) for b in bodies]
    with _engine(cas) as eng:
        for b in bodies[3:]:
            _ingest(eng, b)
    for _ in range(2):
        with _engine(cas) as eng:
            res = {}
            th = [threading.Thread(target=lambda: res.setdefault("imp", eng.import_files(paths))),
                  threading.Thread(target=lambda: res.setdefault("ver", eng.verify(digs[3:])))]
            for t in th:
                t.start()
            for b in bodies[:3]:                                                # a stream publishing the same digests
                assert _ingest(eng, b) == _sha(b)
            for t in th:
                t.join()
            assert res["imp"] == [(DM_OK, d) for d in digs]
            assert all(s == DM_OK for s in res["ver"])
            assert eng.verify(digs) == [DM_OK] * len(digs)
            for d, b in zip(digs, bodies):
                assert eng.fetch(d, chunk=4 << 20) == b.tobytes()
            _clean(eng)
        for d in digs:
            assert _file_hash(_blob_file(cas, d)) == d and os.path.exists(_blob_file(cas, d) + ".meta")
        assert _incoming(cas) == []


def test_live_writers_finish_while_a_large_import_runs(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(900 + i, 3 * SLAB + 5 + i) for i in range(LIVE_FILES)]
    paths = [_write(str(tmp_path / "src" / f"f{i}"), b) for i, b in enumerate(bodies)]
    with _engine(cas, ring_bytes=16 * SLAB) as eng:
        out, done, errors = {}, [], []
        t = threading.Thread(target=lambda: out.setdefault("res", eng.import_files(paths)))

        def writer(k):
            try:
                i = 0
                while t.is_alive() or i == 0:
                    b = _body(5000 + 1000 * k + i, 2 * SLAB + 7 + k)
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
        assert out["res"] == [(DM_OK, _sha(b)) for b in bodies]
        assert len(done) >= 8
        _clean(eng)


def test_the_last_free_stream_slot_stays_with_dm_stream_open(tmp_path):
    from demodel_b200 import DM_ENOMEM, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1200, 1000), _body(1201, 2 * SLAB)]
    paths = [_write(str(tmp_path / "src" / f"f{i}"), b) for i, b in enumerate(bodies)]
    with _engine(cas, max_streams=3) as eng:
        held = [eng.stream_open(None, 0) for _ in range(2)]
        assert eng.import_files(paths) == [(DM_ENOMEM, bytes(32))] * 2          # one slot free: it is not taken
        assert eng.list() == [] and _incoming(cas) == []
        last = eng.stream_open(None, 0)
        for s in held + [last]:
            eng.stream_abort(s)
        assert eng.import_files(paths) == [(DM_OK, _sha(b)) for b in bodies]
        _clean(eng, max_streams=3)


def test_sweep_of_staged_files_left_by_dead_processes(tmp_path):
    cas = str(tmp_path / "cas")
    inc = os.path.join(cas, "incoming")
    os.makedirs(inc)
    gone = subprocess.Popen([sys.executable, "-c", "pass"])
    gone.wait()
    dead = _write(os.path.join(inc, f"{gone.pid}-0-7.part"), b"left by a killed import")
    live = _write(os.path.join(inc, f"{os.getppid()}-0-7.part"), b"another process is still writing this")
    p = _write(str(tmp_path / "src" / "f"), _body(1300, 777))
    with _engine(cas) as eng:
        assert [s for s, _ in eng.import_files([p])] == [0]
        _clean(eng)
    assert not os.path.exists(dead) and os.path.exists(live)


def _ollama_tree(root):
    """A models directory in Ollama's on-disk shape: blobs/sha256-<hex>, manifests/<host>/<ns>/<model>/<tag>."""
    layers = [_body(1400 + i, n) for i, n in enumerate((3 * SLAB + 11, 900, 40000))]
    digs = [_sha(b) for b in layers]
    for d, b in zip(digs, layers):
        _write(os.path.join(root, "blobs", "sha256-" + d.hex()), b)
    manifest = json.dumps({"schemaVersion": 2, "layers": [{"digest": "sha256:" + d.hex(), "size": b.nbytes}
                                                          for d, b in zip(digs, layers)]}).encode()
    _write(os.path.join(root, "manifests", "registry.ollama.ai", "library", "tiny", "latest"), manifest)
    liar = _body(1410, 5000)                                                   # named by another body's digest
    _write(os.path.join(root, "blobs", "sha256-" + _sha(_body(1411, 5000)).hex()), liar)
    partial = _body(1412, 6000)
    _write(os.path.join(root, "blobs", "sha256-" + _sha(partial).hex() + "-partial"), partial)
    return layers, manifest, liar, partial


def _hf_tree(root):
    """A hub cache in HuggingFace's on-disk shape: blobs/, snapshots/<commit>/ links into them, refs/<ref>."""
    weights, config, data = _body(1500, 2 * SLAB + 9), b'{"model_type": "tiny"}', _body(1501, 3000)
    sha1 = hashlib.sha1(b"blob %d\0" % len(config) + config).hexdigest()
    commit = "0123456789abcdef0123456789abcdef01234567"
    repo = os.path.join(root, "models--org--tiny")
    _write(os.path.join(repo, "blobs", _sha(weights).hex()), weights)
    _write(os.path.join(repo, "blobs", sha1), config)
    _write(os.path.join(repo, "blobs", hashlib.sha256(b"x").hexdigest() + ".incomplete"), b"half a download")
    _write(os.path.join(repo, "refs", "main"), commit.encode())
    os.makedirs(os.path.join(repo, "snapshots", commit, "sub"))
    os.symlink(os.path.join("..", "..", "..", "blobs", _sha(weights).hex()),
               os.path.join(repo, "snapshots", commit, "sub", "model.safetensors"))
    os.symlink(os.path.join("..", "..", "blobs", sha1), os.path.join(repo, "snapshots", commit, "config.json"))
    ds = os.path.join(root, "datasets--org--set")
    _write(os.path.join(ds, "blobs", _sha(data).hex()), data)
    _write(os.path.join(ds, "refs", "main"), commit.encode())
    os.makedirs(os.path.join(ds, "snapshots", commit))
    os.symlink(os.path.join("..", "..", "blobs", _sha(data).hex()), os.path.join(ds, "snapshots", commit, "d.parquet"))
    return weights, config, data, commit


def _url_body(eng, url):
    hit = eng.proxy_request(url)
    assert hit is not None, url
    rid, size = hit
    try:
        return eng.cache_read(rid, 0, size) if size else b""
    finally:
        eng.cache_close(rid)


def test_walkers_over_ollama_and_huggingface_trees(tmp_path):
    from demodel_b200 import importer
    cas = str(tmp_path / "cas")
    ollama, hub = str(tmp_path / "ollama"), str(tmp_path / "hub")
    layers, manifest, liar, partial = _ollama_tree(ollama)
    weights, config, data, commit = _hf_tree(hub)
    before = (_tree_state(ollama), _tree_state(hub))
    with _engine(cas) as eng:
        so = importer.import_entries(eng, importer.ollama_entries(ollama), page=2)
        sh = importer.import_entries(eng, importer.hf_entries(hub), link=True)
        assert so["status"] == {"DM_OK": 4, "DM_ECORRUPT": 1} and so["aliases"] == 1
        assert [c["got"] for c in so["corrupt"]] == [_sha(liar).hex()]
        assert sh["status"] == {"DM_OK": 3} and sh["aliases"] == 6 and sh["corrupt"] == []
        for b in layers + [weights, data]:
            assert eng.fetch(_sha(b), chunk=4 << 20) == b.tobytes()
        for b in (liar, partial):
            assert eng.cache_contains(_sha(b)) is None
        assert eng.cache_contains(hashlib.sha256(b"half a download").digest()) is None
        assert _url_body(eng, "https://registry.ollama.ai/v2/library/tiny/manifests/latest") == manifest
        base = "https://huggingface.co/org/tiny/resolve/"
        for rev in (commit, "main"):
            assert _url_body(eng, base + rev + "/config.json") == config
            assert _url_body(eng, base + rev + "/sub/model.safetensors") == weights.tobytes()
            assert _url_body(eng, f"https://huggingface.co/datasets/org/set/resolve/{rev}/d.parquet") == data.tobytes()
        assert _incoming(cas) == []
        _clean(eng)
    assert (_tree_state(ollama), _tree_state(hub)) == before
    tool = _load_tool()                                                         # the command line, in this process
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert tool.main(["--cas-dir", cas, "--hf-cache", hub]) == 0
    summary = json.loads(buf.getvalue())
    assert summary["status"] == {"DM_OK": 3} and summary["aliases"] == 6


def _load_tool():
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "dm_import.py")
    spec = importlib.util.spec_from_file_location("dm_import_tool", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod
