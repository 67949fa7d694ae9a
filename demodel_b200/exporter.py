"""Write cached models out in the layouts importer.py reads (dm_cache_export): the inverse of importer.py.

Two layouts are written:
- an Ollama models directory: every alias ``https://<host>/v2/<ns>/<model>/manifests/<tag>`` (the form importer.py
  enters) names a manifest.  Its config and layers go to ``blobs/sha256-<hex>``, and the manifest itself to
  ``manifests/<host>/<ns>/<model>/<tag>`` last, and only when every blob it lists was exported, so that Ollama never
  sees a manifest whose blobs are missing;
- a HuggingFace hub cache: every alias ``https://huggingface.co/[datasets/|spaces/]<org>/<name>/resolve/<rev>/<path>``
  names a snapshot file.  Blobs go to ``<kind>--<org>--<name>/blobs/<name>``, ``snapshots/<commit>/<path>`` become the
  relative symlinks into ``blobs/`` that huggingface_hub makes, and ``refs/<ref>`` name the commits of non-hex
  revisions.

Only the alias index and the blobs' sidecars are read; nothing is hashed on the CPU.  Every byte written is hashed on
the GPU by dm_cache_export before it is renamed into place.
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass, field
from typing import Iterable, Optional
from urllib.parse import unquote

from ._lib import DM_OK, DmError
from .importer import HF_ENDPOINT, _HEX40
from .manifest import parse_manifest

_OLLAMA_KEY = re.compile(r"https://([^/]+)/v2/([^/]+)/([^/]+)/manifests/([^/]+)")
_HF_KEY = re.compile(re.escape(HF_ENDPOINT) + r"/(?:(datasets|spaces)/)?([^/]+)/([^/]+)/resolve/([^/]+)/(.+)")


@dataclass
class Export:
    digest: bytes
    path: str


@dataclass
class Plan:
    """What to write, in order: blobs first; then each manifest whose blobs (indices into ``blobs``) all ended DM_OK;
    then each symlink whose blob did; then the refs.  ``skipped`` lists what cannot be exported, with the reason."""
    blobs: list[Export] = field(default_factory=list)
    manifests: list[tuple[Export, list[int]]] = field(default_factory=list)
    links: list[tuple[str, int]] = field(default_factory=list)        # (snapshot path, index of its blob)
    refs: dict[str, str] = field(default_factory=dict)                # refs/<ref> file -> commit
    skipped: list[dict] = field(default_factory=list)
    _index: dict[str, int] = field(default_factory=dict)

    def blob(self, digest: bytes, path: str) -> Optional[int]:
        """Index of the blob export to `path`; None when `path` is already planned with another digest."""
        k = self._index.get(path)
        if k is None:
            k = self._index[path] = len(self.blobs)
            self.blobs.append(Export(digest, path))
        return k if self.blobs[k].digest == digest else None


def _wanted(only: Optional[Iterable[str]], names: list[str]) -> bool:
    return only is None or any(n in only for n in names)


def _read_verified(eng, digest: bytes) -> Optional[bytes]:
    """The whole blob, read through a verified ring open (no HBM extent taken); None when it is not cached."""
    opened = eng.cache_open_verified_ring(digest)
    if opened is None:
        return None
    rid, size = opened
    try:
        parts, off = [], 0
        while off < size:
            part = eng.cache_read(rid, off, min(1 << 20, size - off))
            if not part:
                break
            parts.append(part)
            off += len(part)
        return b"".join(parts)
    finally:
        eng.cache_close(rid)


def _headers(eng, digest: bytes) -> dict[str, str]:
    """The response headers the blob's sidecar recorded, names lower-cased ({} without a sidecar)."""
    if not getattr(eng, "cas_dir", None):
        return {}
    h = digest.hex()
    try:
        with open(os.path.join(eng.cas_dir, "blobs", "sha256", h[:2], h + ".meta")) as f:
            meta = json.load(f)
    except (OSError, ValueError):
        return {}
    headers = meta.get("headers") if isinstance(meta, dict) else None
    return {str(k).lower(): str(v) for k, v in headers.items()} if isinstance(headers, dict) else {}


def ollama_plan(eng, models_dir: str, only: Optional[Iterable[str]] = None) -> Plan:
    """Every manifest alias of the engine, as an Ollama models directory under `models_dir`.  `only`: names to keep,
    each ``<model>``, ``<model>:<tag>``, ``<ns>/<model>``, ``<ns>/<model>:<tag>`` or ``<host>/<ns>/<model>:<tag>``."""
    only = set(only) if only is not None else None
    plan = Plan()
    for key, digest in eng.alias_list("https://"):
        m = _OLLAMA_KEY.fullmatch(key)
        if not m:
            continue
        host, ns, model, tag = m.groups()
        if not _wanted(only, [model, f"{model}:{tag}", f"{ns}/{model}", f"{ns}/{model}:{tag}",
                              f"{host}/{ns}/{model}:{tag}"]):
            continue
        try:
            body = _read_verified(eng, digest)
        except DmError as ex:
            plan.skipped.append({"key": key, "why": f"the manifest could not be read: {ex}"})
            continue
        if body is None:
            plan.skipped.append({"key": key, "why": "the manifest is not cached"})
            continue
        try:
            layers = parse_manifest(body)
        except DmError:
            plan.skipped.append({"key": key, "why": "not an image manifest"})
            continue
        needs = [plan.blob(l.digest, os.path.join(models_dir, "blobs", "sha256-" + l.digest.hex())) for l in layers]
        plan.manifests.append((Export(digest, os.path.join(models_dir, "manifests", host, ns, model, tag)), needs))
    return plan


def hf_plan(eng, hub_dir: str, only: Optional[Iterable[str]] = None) -> Plan:
    """Every resolve/ alias of the engine, as a HuggingFace hub cache under `hub_dir`.  `only`: repository ids to keep
    (``<org>/<name>``, ``datasets/<org>/<name>``, ``spaces/<org>/<name>``).

    A file's commit is its revision when that is 40 hex digits, else the X-Repo-Commit header its sidecar recorded,
    else the one commit whose resolve/<commit>/ aliases give every file under that revision the same digests.  A blob is
    named by its ETag when that is a git blob id (40 hex digits), else by its SHA-256."""
    only = set(only) if only is not None else None
    files: dict[str, dict[str, dict[str, bytes]]] = {}      # repo dir -> revision -> path -> digest
    for key, digest in eng.alias_list(HF_ENDPOINT + "/"):
        m = _HF_KEY.fullmatch(key)
        if not m:
            continue
        kind, org, name, rev, path = m.groups()
        if not _wanted(only, [f"{org}/{name}", f"{kind or 'models'}/{org}/{name}", f"{kind}/{org}/{name}"]):
            continue
        repo = f"{kind or 'models'}--{org}--{name}"
        files.setdefault(repo, {}).setdefault(unquote(rev), {})[unquote(path)] = digest
    plan = Plan()
    for repo, revs in sorted(files.items()):
        repo_dir = os.path.join(hub_dir, repo)
        commits = {r: t for r, t in revs.items() if _HEX40.fullmatch(r)}
        ref_commit: dict[str, Optional[str]] = {}            # non-hex revision -> commit (None: the files disagree)
        snaps: dict[tuple[str, str], bytes] = {}             # (commit, path) -> digest
        for rev, tree in sorted(revs.items()):
            inferred = [c for c, t in sorted(commits.items()) if t == tree] if rev not in commits else []
            for path, digest in sorted(tree.items()):
                if rev in commits:
                    commit = rev
                else:
                    commit = _headers(eng, digest).get("x-repo-commit", "").strip().lower()
                    if not _HEX40.fullmatch(commit):
                        commit = inferred[0] if len(inferred) == 1 else ""
                    if not commit:
                        plan.skipped.append({"key": f"{repo}/{rev}/{path}",
                                             "why": "no commit: the revision is not a commit id, the sidecar records no "
                                                    "X-Repo-Commit, and no single cached commit has the same files"})
                        continue
                    seen = ref_commit.setdefault(rev, commit)
                    if seen is not None and seen != commit:
                        ref_commit[rev] = None
                if snaps.setdefault((commit, path), digest) != digest:
                    plan.skipped.append({"key": f"{repo}/{commit}/{path}", "why": "two digests for one snapshot file"})
        for (commit, path), digest in sorted(snaps.items()):
            etag = _headers(eng, digest).get("etag", "").strip()
            etag = etag[2:] if etag.startswith("W/") else etag
            etag = etag.strip('"').lower()
            blob_name = etag if _HEX40.fullmatch(etag) else digest.hex()
            k = plan.blob(digest, os.path.join(repo_dir, "blobs", blob_name))
            if k is None:
                plan.skipped.append({"key": f"{repo}/{commit}/{path}", "why": f"blob name {blob_name} names another digest"})
                continue
            plan.links.append((os.path.join(repo_dir, "snapshots", commit, *path.split("/")), k))
        for rev, commit in sorted(ref_commit.items()):
            if commit is None:
                plan.skipped.append({"key": f"{repo}/refs/{rev}", "why": "its files disagree about which commit it names"})
            else:
                plan.refs[os.path.join(repo_dir, "refs", *rev.split("/"))] = commit
    return plan


def _replace(path: str, make) -> None:
    """Create `path` through a temporary name next to it and a rename: readers never see half of it."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    tmp = os.path.join(os.path.dirname(path), f".{os.path.basename(path)}.dm-export-{os.getpid()}.tmp")
    try:
        os.unlink(tmp)
    except FileNotFoundError:
        pass
    make(tmp)
    os.replace(tmp, path)


def _write_ref(tmp: str, commit: str) -> None:
    with open(tmp, "w") as f:
        f.write(commit)


def export_entries(eng, plan: Plan, page: int = 1024) -> dict:
    """Carry out `plan` through ``eng.export`` in pages of `page` files.  Returns a summary: counts per status name,
    bytes exported, the entries whose copy did not hash to its name, and what was skipped and why."""
    from . import _lib
    names = {getattr(_lib, n): n for n in dir(_lib) if n.startswith("DM_E") or n == "DM_OK"}
    summary = {"status": {}, "bytes_exported": 0, "corrupt": [], "skipped": list(plan.skipped), "links": 0, "refs": 0}

    def run(items: list[Export]) -> list[int]:
        out = []
        for i in range(0, len(items), page):
            chunk = items[i:i + page]
            res = eng.export([x.digest for x in chunk], [x.path for x in chunk])
            for x, st in zip(chunk, res):
                name = names.get(st, str(st))
                summary["status"][name] = summary["status"].get(name, 0) + 1
                if st == DM_OK:
                    summary["bytes_exported"] += os.path.getsize(x.path)
                elif name == "DM_ECORRUPT":
                    summary["corrupt"].append({"digest": x.digest.hex(), "path": x.path})
                elif name == "DM_ENOENT":
                    summary["skipped"].append({"key": x.path, "why": f"sha256:{x.digest.hex()} is not cached"})
            out += res
        return out

    ok = [st == DM_OK for st in run(plan.blobs)]
    ready = []
    for m, needs in plan.manifests:
        if all(ok[k] for k in needs):
            ready.append(m)
        else:
            summary["skipped"].append({"key": m.path, "why": "a blob it lists was not exported"})
    run(ready)
    for link, k in plan.links:
        if not ok[k]:
            summary["skipped"].append({"key": link, "why": "its blob was not exported"})
            continue
        target = os.path.relpath(plan.blobs[k].path, os.path.dirname(link))
        _replace(link, lambda tmp: os.symlink(target, tmp))
        summary["links"] += 1
    for ref, commit in sorted(plan.refs.items()):
        _replace(ref, lambda tmp: _write_ref(tmp, commit))
        summary["refs"] += 1
    return summary
