"""dm_cache_export on the GPU: cached blobs are copied to a private file next to their destination (out of HBM, or from
the disk tier), hashed there by the SHA-256 kernels with the digest as the expected value, and renamed over the
destination only on a match.  The cache is only read.  Every file written is checked against hashlib.

Sizes are module constants so that tests/test_export_host.py can run the same tests over the fake CUDA runtime with a
small ring and arena."""
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

ARENA = 512 << 20           # HBM arena of the exporting engines
RING = 64 << 20
SLAB = 1 << 20
SMALL_ARENA = 16 << 20      # the arena of the DM_F_NO_HBM_CAS engine a large blob is exported from
BIG = 96 << 20              # a large layer; also the blob held while dm_cache_remove and a disk limit race the export
LARGE = 160 << 20           # larger than both the ring and SMALL_ARENA
MANY = 3000                 # tiny files (at most 8 KiB) in one call
LIVE = 8                    # writers streaming bodies while a large export runs


def _body(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _sha(body):
    return hashlib.sha256(body.tobytes() if isinstance(body, np.ndarray) else body).digest()


def _engine(cas, hbm=None, **kw):
    import demodel_b200
    kw.setdefault("ring_bytes", RING)
    return demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA if hbm is None else hbm, slab_bytes=SLAB, cas_dir=cas,
                               **kw)


def _write(path, body):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(body.tobytes() if isinstance(body, np.ndarray) else body)
    return path


def _blob_file(cas, dig):
    return os.path.join(cas, "blobs", "sha256", dig.hex()[:2], dig.hex())


def _file_hash(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 24), b""):
            h.update(chunk)
    return h.digest()


def _ingest(eng, body):
    sid = eng.stream_open(_sha(body), body.nbytes)
    for off in range(0, body.nbytes, 1 << 20):
        eng.stream_write(sid, body[off:off + (1 << 20)])
    dig, ok = eng.stream_finish(sid)
    assert ok and dig == _sha(body)
    return dig


def _on_disk(eng, tmp_path, bodies, tag="src"):
    """Place bodies in the disk tier only (dm_cache_import never touches HBM)."""
    from demodel_b200 import DM_OK
    paths = [_write(str(tmp_path / tag / f"f{i}"), b) for i, b in enumerate(bodies)]
    digs = [_sha(b) for b in bodies]
    assert eng.import_files(paths, expect=digs) == [(DM_OK, d) for d in digs]
    return digs


def _staged(root):
    """Staged export files left anywhere under root."""
    return [os.path.join(d, f) for d, _, fs in os.walk(root) for f in fs if ".dm-export-" in f]


def _clean(eng, max_streams=65536):
    for _ in range(400):
        st = eng.stats()
        if (st["ring_slabs_free"] == st["ring_slabs_total"] and st["free_stream_slots"] == max_streams
                and st["open_streams"] == 0 and st["open_readers"] == 0):
            return
        time.sleep(0.01)
    raise AssertionError(f"engine not clean: {st}")


def _wait_for(pred, what, timeout=120.0):
    t0 = time.time()
    while not pred():
        if time.time() - t0 > timeout:
            raise AssertionError(f"timed out waiting for {what}")
        time.sleep(0.001)


# ---- layouts ------------------------------------------------------------------------------------------------------

def _hf_hub(root):
    """A hub cache in HuggingFace's shape: LFS blobs named by SHA-256, git files by their git blob id, two commits
    sharing a file, refs/main and refs/pr/1, and a nested sub/dir/ path."""
    weights, shared, sub = _body(100, 2 * SLAB + 9), _body(101, 70000), _body(102, 3000)
    config1, config2 = b'{"model_type": "tiny", "v": 1}', b'{"model_type": "tiny", "v": 2}'
    c1, c2 = "1" * 40, "2" * 40
    repo = os.path.join(root, "models--org--tiny")

    def git_name(b):
        return hashlib.sha1(b"blob %d\0" % len(b) + b).hexdigest()

    names = {}
    for b in (weights, shared, sub):
        names[id(b)] = _sha(b).hex()
        _write(os.path.join(repo, "blobs", names[id(b)]), b)
    for b in (config1, config2):
        names[id(b)] = git_name(b)
        _write(os.path.join(repo, "blobs", names[id(b)]), b)
    trees = {c1: {"config.json": config1, "model.safetensors": weights, "shared.bin": shared},
             c2: {"config.json": config2, "shared.bin": shared, "sub/dir/extra.bin": sub}}
    for commit, tree in trees.items():
        for path, b in tree.items():
            link = os.path.join(repo, "snapshots", commit, *path.split("/"))
            os.makedirs(os.path.dirname(link), exist_ok=True)
            os.symlink(os.path.relpath(os.path.join(repo, "blobs", names[id(b)]), os.path.dirname(link)), link)
    _write(os.path.join(repo, "refs", "main"), c2.encode())
    _write(os.path.join(repo, "refs", "pr", "1"), c1.encode())
    return repo, trees


def _snapshot_bytes(repo):
    out = {}
    snaps = os.path.join(repo, "snapshots")
    for d, _, fs in os.walk(snaps):
        for f in fs:
            p = os.path.join(d, f)
            assert os.path.islink(p), p
            with open(p, "rb") as fh:
                out[os.path.relpath(p, snaps)] = fh.read()
    return out


def _refs(repo):
    out = {}
    for d, _, fs in os.walk(os.path.join(repo, "refs")):
        for f in fs:
            with open(os.path.join(d, f)) as fh:
                out[os.path.relpath(os.path.join(d, f), os.path.join(repo, "refs"))] = fh.read()
    return out


def test_huggingface_round_trip_from_the_disk_tier(tmp_path):
    from demodel_b200 import exporter, importer
    hub, out = str(tmp_path / "hub"), str(tmp_path / "out")
    cas1, cas3 = str(tmp_path / "cas1"), str(tmp_path / "cas3")
    repo, trees = _hf_hub(hub)
    with _engine(cas1) as eng:
        s = importer.import_entries(eng, importer.hf_entries(hub))
        assert s["corrupt"] == [] and set(s["status"]) == {"DM_OK"}
        aliases1 = dict(eng.alias_list(importer.HF_ENDPOINT))
    with _engine(cas1) as eng:                                    # restarted: every blob is on the disk tier only
        st0 = eng.stats()
        plan = exporter.hf_plan(eng, out)
        summary = exporter.export_entries(eng, plan)
        st = eng.stats()
        assert summary["corrupt"] == [] and summary["skipped"] == [], summary
        assert set(summary["status"]) == {"DM_OK"} and summary["refs"] == 2
        assert st["hbm_cas_used"] == st0["hbm_cas_used"] and st["d2h_bytes"] == st0["d2h_bytes"]
        _clean(eng)
    orepo = os.path.join(out, "models--org--tiny")
    assert _snapshot_bytes(orepo) == _snapshot_bytes(repo)
    assert _refs(orepo) == _refs(repo)
    lfs = lambda r: sorted(n for n in os.listdir(os.path.join(r, "blobs")) if len(n) == 64)
    assert set(lfs(repo)) <= set(lfs(orepo))                      # git files without an ETag are named by SHA-256
    for d, _, fs in os.walk(os.path.join(orepo, "snapshots")):
        for f in fs:
            target = os.readlink(os.path.join(d, f))
            assert not os.path.isabs(target) and target.startswith("../../") and "/blobs/" in "/" + target
    assert _staged(out) == []
    with _engine(cas3) as eng:
        s = importer.import_entries(eng, importer.hf_entries(out))
        assert s["corrupt"] == [] and set(s["status"]) == {"DM_OK"}
        assert dict(eng.alias_list(importer.HF_ENDPOINT)) == aliases1


def _ollama_models(root):
    config = json.dumps({"model_format": "gguf", "model_family": "tiny"}).encode()
    big, license_ = _body(200, BIG + 13), b"Apache License 2.0\n" * 2000            # license: at most 64 KiB
    assert len(license_) <= 64 << 10
    parts = [config, big, license_]
    for b in parts:
        _write(os.path.join(root, "blobs", "sha256-" + _sha(b).hex()), b)
    manifest = json.dumps({"schemaVersion": 2, "mediaType": "application/vnd.docker.distribution.manifest.v2+json",
                           "config": {"digest": "sha256:" + _sha(config).hex(), "size": len(config)},
                           "layers": [{"digest": "sha256:" + _sha(b).hex(), "size": len(b)} for b in parts[1:]]}).encode()
    _write(os.path.join(root, "manifests", "registry.ollama.ai", "library", "tiny", "latest"), manifest)
    return parts, manifest


def _tree_bytes(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            with open(os.path.join(d, f), "rb") as fh:
                out[os.path.relpath(os.path.join(d, f), root)] = hashlib.sha256(fh.read()).hexdigest()
    return out


def test_ollama_round_trip_and_no_manifest_without_its_blobs(tmp_path):
    from demodel_b200 import DM_OK, exporter, importer
    models, out, out2 = str(tmp_path / "models"), str(tmp_path / "out"), str(tmp_path / "out2")
    cas = str(tmp_path / "cas")
    parts, manifest = _ollama_models(models)
    with _engine(cas) as eng:
        s = importer.import_entries(eng, importer.ollama_entries(models))
        assert s["status"] == {"DM_OK": 4}
    with _engine(cas) as eng:
        summary = exporter.export_entries(eng, exporter.ollama_plan(eng, out))
        assert summary["status"] == {"DM_OK": 4} and summary["corrupt"] == [] and summary["skipped"] == []
        assert summary["bytes_exported"] == sum(len(b) for b in parts) + len(manifest)
        assert _tree_bytes(out) == _tree_bytes(models)
        assert exporter.ollama_plan(eng, out2, only=["library/other"]).manifests == []
        assert eng.cache_remove([_sha(parts[2])]) == [DM_OK]           # a layer leaves the cache
        summary = exporter.export_entries(eng, exporter.ollama_plan(eng, out2, only=["tiny"]))
        assert summary["status"] == {"DM_OK": 2, "DM_ENOENT": 1}
        assert not os.path.exists(os.path.join(out2, "manifests"))    # Ollama never sees a manifest without its blobs
        assert any("manifests" in s["key"] for s in summary["skipped"])
        _clean(eng)
    assert _staged(out) == [] and _staged(out2) == []


# ---- the engine call ------------------------------------------------------------------------------------------------

def test_from_hbm_without_a_cas_dir(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_OK
    bodies = [_body(300 + i, n) for i, n in enumerate((0, 1, 4097, 64 << 10, (64 << 10) + 1, 3 * SLAB + 5))]
    with demodel_b200.Engine(device=0, hbm_cas_bytes=ARENA, ring_bytes=RING, slab_bytes=SLAB) as eng:
        digs = [_ingest(eng, b) for b in bodies]
        st0 = eng.stats()
        dests = [str(tmp_path / "out" / "deep" / f"f{i}") for i in range(len(bodies))]
        assert eng.export(digs, dests) == [DM_OK] * len(bodies)
        st = eng.stats()
        total = sum(b.nbytes for b in bodies)
        assert st["d2h_bytes"] - st0["d2h_bytes"] == total
        assert st["bytes_hashed"] - st0["bytes_hashed"] == total
        assert st["h2d_bytes"] - st0["h2d_bytes"] == total
        assert st["hbm_cas_used"] == st0["hbm_cas_used"] and st["bytes_served"] == st0["bytes_served"]
        for k in ("blobs_committed", "blobs_mismatched", "bytes_ingested"):
            assert st[k] == st0[k], k
        for d, p, b in zip(digs, dests, bodies):
            assert _file_hash(p) == d and os.path.getsize(p) == b.nbytes
        # the LRU order is untouched: fill the arena and the blob that was least recently used before the export is
        # still the first to go
        first, second = digs[-1], _ingest(eng, _body(399, 3 * SLAB + 5))
        assert eng.export([first], [str(tmp_path / "again")]) == [DM_OK]
        k = 0
        while eng.cache_contains(first) is not None:                    # (one ingest may evict both at once)
            _ingest(eng, _body(5000 + k, 4 * SLAB))
            k += 1
            assert k < 4 * ARENA // (4 * SLAB)
            assert not (eng.cache_contains(second) is None and eng.cache_contains(first) is not None)
        assert _staged(str(tmp_path)) == []
        _clean(eng)


def test_corrupt_tier_file_is_never_written_and_is_left_to_verify(tmp_path):
    from demodel_b200 import DM_ECORRUPT, DM_ENOENT, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(400, 3 * SLAB + 17), _body(401, 5000), _body(402, 2 * SLAB)]
    with _engine(cas) as eng:
        digs = _on_disk(eng, tmp_path, bodies)
    flip = [_blob_file(cas, d) for d in digs[:2]]
    for p in flip:                                                      # one byte flipped in place
        with open(p, "r+b") as f:
            f.seek(os.path.getsize(p) // 2)
            b = f.read(1)
            f.seek(-1, 1)
            f.write(bytes([b[0] ^ 0x40]))
    with open(_blob_file(cas, digs[2]), "ab") as f:                    # size no longer its sidecar's
        f.write(b"x")
    before = {p: (_file_hash(p), os.stat(p).st_mtime_ns) for p in map(lambda d: _blob_file(cas, d), digs)}
    with _engine(cas) as eng:
        dests = [str(tmp_path / "out" / f"f{i}") for i in range(3)]
        assert eng.export(digs, dests) == [DM_ECORRUPT] * 3
        assert "dm_cache_verify" in eng.error_detail(0)
        assert not any(os.path.exists(p) for p in dests) and _staged(str(tmp_path / "out")) == []
        assert {p: (_file_hash(p), os.stat(p).st_mtime_ns) for p in before} == before
        assert eng.verify(digs) == [DM_ECORRUPT] * 3                    # verify decides: the files go
        assert not any(os.path.exists(p) for p in before)
        assert eng.export(digs, dests) == [DM_ENOENT] * 3
        _clean(eng)


def test_statuses_duplicates_and_atomic_replace(tmp_path):
    import demodel_b200
    from demodel_b200 import DM_EINVAL, DM_ENOENT, DM_EIO, DM_OK
    cas = str(tmp_path / "cas")
    a, b = _body(500, 2 * SLAB + 3), _body(501, 700)
    out = tmp_path / "out"
    with _engine(cas) as eng:
        da, db = _on_disk(eng, tmp_path, [a, b])
        missing = _sha(b"not cached")
        os.makedirs(out / "adir")
        old = _write(str(out / "replace"), b"the old bytes")
        fd = os.open(old, os.O_RDONLY)
        try:
            st0 = eng.stats()
            dests = [str(out / "a"), str(out / "missing"), str(out / "adir"), str(out / "a"), str(out / "b"),
                     str(out / "replace")]
            res = eng.export([da, missing, da, da, db, db], dests)
            assert res == [DM_OK, DM_ENOENT, DM_EIO, DM_OK, DM_OK, DM_OK]
            assert eng.stats()["bytes_hashed"] - st0["bytes_hashed"] == a.nbytes + 2 * b.nbytes   # duplicates once
            assert os.pread(fd, 100, 0) == b"the old bytes"             # the old file lives on for its reader
        finally:
            os.close(fd)
        assert _file_hash(str(out / "replace")) == db and _file_hash(str(out / "a")) == da
        assert os.path.isdir(out / "adir")
        with pytest.raises(demodel_b200.DmError) as ex:
            eng.export([da, db], [str(out / "x"), str(out / "x")])
        assert ex.value.code == DM_EINVAL and not os.path.exists(out / "x")
        assert eng.export([], []) == []
        assert _staged(str(out)) == []
        _clean(eng)


def test_large_blob_on_an_engine_without_an_hbm_tier(tmp_path):
    from demodel_b200 import DM_OK
    from demodel_b200._lib import DM_F_NO_HBM_CAS
    cas = str(tmp_path / "cas")
    body = _body(600, LARGE + 65)
    assert body.nbytes > RING and body.nbytes > SMALL_ARENA
    with _engine(cas, hbm=SMALL_ARENA, flags=DM_F_NO_HBM_CAS) as eng:
        (d,) = _on_disk(eng, tmp_path, [body])
        st0 = eng.stats()
        assert eng.export([d], [str(tmp_path / "out" / "large")]) == [DM_OK]
        st = eng.stats()
        assert st["bytes_hashed"] - st0["bytes_hashed"] == body.nbytes and st["d2h_bytes"] == st0["d2h_bytes"]
        assert _file_hash(str(tmp_path / "out" / "large")) == d
        _clean(eng)


def test_many_tiny_files_share_launches(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    rng = np.random.default_rng(700)
    bodies = [rng.integers(0, 256, int(n), dtype=np.uint8) for n in rng.integers(1, 8192, MANY)]
    with _engine(cas) as eng:
        digs = _on_disk(eng, tmp_path, bodies)
        st0 = eng.stats()
        dests = [str(tmp_path / "out" / f"{i % 7}" / f"{i:05d}") for i in range(MANY)]
        assert eng.export(digs, dests) == [DM_OK] * MANY
        st = eng.stats()
        assert st["packed_bodies"] - st0["packed_bodies"] >= MANY // 2              # (a pack may be full for a moment)
        assert st["kernel_launches"] - st0["kernel_launches"] < MANY // 10          # the chains went out together
        assert st["bytes_hashed"] - st0["bytes_hashed"] == sum(b.nbytes for b in bodies)
        for d, p in zip(digs[::97], dests[::97]):
            assert _file_hash(p) == d
        _clean(eng)


def _export_in_thread(eng, digs, dests):
    out = {}
    t = threading.Thread(target=lambda: out.setdefault("res", eng.export(digs, dests)))
    t.start()
    return t, out


def test_remove_and_a_tight_disk_limit_during_an_export(tmp_path):
    from demodel_b200 import DM_ENOENT, DM_ESTATE, DM_OK
    cas = str(tmp_path / "cas")
    big, other = _body(800, BIG + 1), _body(801, 3 * SLAB)
    out = str(tmp_path / "out")
    with _engine(cas) as eng:
        d, d_other = _on_disk(eng, tmp_path, [big, other])
        t, res = _export_in_thread(eng, [d], [os.path.join(out, "big")])
        _wait_for(lambda: _staged(out) or not t.is_alive(), "the staged file")
        part = _staged(out)
        st = eng.cache_remove([d])
        assert st == [DM_ESTATE] or not any(os.path.exists(p) for p in part)
        eng.set_disk_limit(1)                                           # every blob is a victim, but a pinned one
        t.join()
        assert res["res"] == [DM_OK] and _file_hash(os.path.join(out, "big")) == d
        assert not os.path.exists(_blob_file(cas, d_other))            # the limit did evict what it could
        eng.set_disk_limit(0)
        assert eng.cache_remove([d]) in ([DM_OK], [DM_ENOENT])          # after the verdict it runs
        assert _staged(out) == []
        _clean(eng)


def test_streams_opened_during_a_large_export_finish(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(900 + i, 3 * SLAB + 7 + i) for i in range(8)]
    out = str(tmp_path / "out")
    with _engine(cas, ring_bytes=16 * SLAB) as eng:
        digs = _on_disk(eng, tmp_path, bodies)
        t, res = _export_in_thread(eng, digs, [os.path.join(out, f"f{i}") for i in range(len(digs))])
        done, errors = [], []

        def writer(k):
            try:
                i = 0
                while t.is_alive() or i == 0:
                    b = _body(5000 + 1000 * k + i, 2 * SLAB + 7 + k)
                    assert _ingest(eng, b) == _sha(b)
                    done.append(1)
                    i += 1
            except Exception as ex:                                    # reported by the main thread
                errors.append(ex)
        ws = [threading.Thread(target=writer, args=(k,)) for k in range(LIVE)]
        for w in ws:
            w.start()
        t.join()
        for w in ws:
            w.join()
        assert not errors, errors
        assert res["res"] == [DM_OK] * len(digs) and len(done) >= LIVE
        for i, d in enumerate(digs):
            assert _file_hash(os.path.join(out, f"f{i}")) == d
        _clean(eng)


def test_the_cache_is_unchanged_by_exports(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1000 + i, n) for i, n in enumerate((10, 5000, 2 * SLAB + 1, SLAB + 3))]
    with _engine(cas) as eng:
        digs = _on_disk(eng, tmp_path, bodies)
        eng.set_disk_limit(1 << 40)
        assert eng.promote(digs[-1:]) == [DM_OK]                        # one of them in HBM as well
        files = [_blob_file(cas, d) for d in digs]
        mtimes = [os.stat(p).st_mtime_ns for p in files]
        st0, du0 = eng.stats(), eng.disk_usage()
        for _ in range(2):
            assert eng.export(digs, [str(tmp_path / "out" / f"f{i}") for i in range(4)]) == [DM_OK] * 4
        st, du = eng.stats(), eng.disk_usage()
        assert st["d2h_bytes"] - st0["d2h_bytes"] == 2 * bodies[-1].nbytes
        for k in ("blobs_committed", "blobs_mismatched", "bytes_ingested", "hbm_cas_used"):
            assert st[k] == st0[k], k
        assert du == du0
        assert [os.stat(p).st_mtime_ns for p in files] == mtimes          # an export is not a use
        _clean(eng)


def test_the_last_free_stream_slot_stays_with_dm_stream_open(tmp_path):
    from demodel_b200 import DM_ENOMEM, DM_OK
    cas = str(tmp_path / "cas")
    bodies = [_body(1150, 1000), _body(1151, 2 * SLAB)]
    out = tmp_path / "out"
    dests = [str(out / f"f{i}") for i in range(len(bodies))]
    with _engine(cas, max_streams=3) as eng:
        digs = _on_disk(eng, tmp_path, bodies)
        held = [eng.stream_open(None, 0) for _ in range(2)]
        assert eng.export(digs, dests) == [DM_ENOMEM, DM_ENOMEM]                # one slot free: it is not taken
        assert not any(os.path.exists(p) for p in dests) and _staged(str(out)) == []
        last = eng.stream_open(None, 0)
        for s in held + [last]:
            eng.stream_abort(s)
        assert eng.export(digs, dests) == [DM_OK, DM_OK]
        for d, p in zip(digs, dests):
            assert _file_hash(p) == d
        _clean(eng, max_streams=3)


def test_stale_staging_files_of_dead_processes_are_swept(tmp_path):
    from demodel_b200 import DM_OK
    cas = str(tmp_path / "cas")
    out = tmp_path / "out"
    gone = subprocess.Popen([sys.executable, "-c", "pass"])
    gone.wait()
    dead = _write(str(out / f".model.bin.dm-export-{gone.pid}-7.part"), b"left by a killed export")
    live = _write(str(out / f".model.bin.dm-export-{os.getppid()}-7.part"), b"another process is still writing this")
    elsewhere = _write(str(tmp_path / "other" / f".x.dm-export-{gone.pid}-7.part"), b"not a directory it writes to")
    with _engine(cas) as eng:
        (d,) = _on_disk(eng, tmp_path, [_body(1100, 777)])
        assert eng.export([d], [str(out / "model.bin")]) == [DM_OK]
        _clean(eng)
    assert not os.path.exists(dead) and os.path.exists(live) and os.path.exists(elsewhere)


def test_command_line_writes_a_hub_cache(tmp_path):
    import contextlib
    import importlib.util
    import io
    from demodel_b200 import importer
    hub, out, cas = str(tmp_path / "hub"), str(tmp_path / "out"), str(tmp_path / "cas")
    repo, _ = _hf_hub(hub)
    with _engine(cas) as eng:
        assert importer.import_entries(eng, importer.hf_entries(hub))["corrupt"] == []
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "dm_export.py")
    spec = importlib.util.spec_from_file_location("dm_export_tool", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert tool.main(["--cas-dir", cas, "--hf-cache", out, "--only", "org/other"]) == 0
    assert json.loads(buf.getvalue())["status"] == {} and not os.path.exists(out)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert tool.main(["--cas-dir", cas, "--hf-cache", out, "--only", "org/tiny"]) == 0
    summary = json.loads(buf.getvalue())
    assert set(summary["status"]) == {"DM_OK"} and summary["refs"] == 2 and summary["destination"] == out
    assert _snapshot_bytes(os.path.join(out, "models--org--tiny")) == _snapshot_bytes(repo)
