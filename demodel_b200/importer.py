"""Seed the disk tier from the layouts that hold models on a host (dm_cache_import).

Two layouts are walked:
- an Ollama models directory (``~/.ollama/models``): ``blobs/sha256-<hex>`` named by their SHA-256, and
  ``manifests/<host>/<namespace>/<model>/<tag>``, which are entered under the registry URL the client asks for;
- a HuggingFace hub cache (``~/.cache/huggingface/hub``): ``models--<org>--<name>`` (also ``datasets--`` and
  ``spaces--``) with ``blobs/`` (LFS files named by their SHA-256, regular files by their git SHA-1),
  ``snapshots/<commit>/<path>`` symlinks into ``blobs/`` and ``refs/<ref>`` files naming a commit.  Every snapshot
  path is entered under its ``resolve/<commit>/`` URL and under ``resolve/<ref>/`` for each ref naming that commit,
  the URL form the proxy's body tee records.

The walkers only read the directories they are given; the engine hashes every file on the GPU.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Iterator, Optional
from urllib.parse import quote

from ._lib import DM_OK

_HEX64 = re.compile(r"[0-9a-f]{64}")
_HEX40 = re.compile(r"[0-9a-f]{40}")
HF_ENDPOINT = "https://huggingface.co"
_HF_KINDS = {"models": "", "datasets": "datasets/", "spaces": "spaces/"}


@dataclass
class Entry:
    path: str                       # the file to import
    expect: Optional[bytes]         # its SHA-256 when the layout names it
    keys: list[str]                 # URLs to enter in the alias index once it is cached


def ollama_entries(models_dir: str) -> Iterator[Entry]:
    """Blobs (``sha256-<hex>``, partial downloads skipped) and manifests of an Ollama models directory."""
    blobs = os.path.join(models_dir, "blobs")
    if os.path.isdir(blobs):
        for name in sorted(os.listdir(blobs)):
            if "-partial" in name or not name.startswith("sha256-") or not _HEX64.fullmatch(name[7:]):
                continue
            yield Entry(os.path.join(blobs, name), bytes.fromhex(name[7:]), [])
    manifests = os.path.join(models_dir, "manifests")
    for dirpath, dirnames, filenames in os.walk(manifests):
        dirnames.sort()
        rel = os.path.relpath(dirpath, manifests).split(os.sep)
        if len(rel) != 3:                                     # <host>/<namespace>/<model>
            continue
        host, namespace, model = rel
        for tag in sorted(filenames):
            yield Entry(os.path.join(dirpath, tag), None, [f"https://{host}/v2/{namespace}/{model}/manifests/{tag}"])


def _read_refs(repo_dir: str) -> dict[str, list[str]]:
    """commit -> the refs naming it (``main``, ``refs/pr/1`` ...)."""
    out: dict[str, list[str]] = {}
    refs = os.path.join(repo_dir, "refs")
    for dirpath, dirnames, filenames in os.walk(refs):
        dirnames.sort()
        for f in sorted(filenames):
            p = os.path.join(dirpath, f)
            try:
                with open(p) as fh:
                    commit = fh.read().strip()
            except OSError:
                continue
            out.setdefault(commit, []).append(os.path.relpath(p, refs).replace(os.sep, "/"))
    return out


def hf_entries(hub_dir: str) -> Iterator[Entry]:
    """Blobs of every repository of a HuggingFace hub cache, each with the resolve/ URLs its snapshots give it."""
    for repo in sorted(os.listdir(hub_dir)):
        kind, sep, rest = repo.partition("--")
        repo_dir = os.path.join(hub_dir, repo)
        if not sep or kind not in _HF_KINDS or not rest or not os.path.isdir(repo_dir):
            continue
        base = f"{HF_ENDPOINT}/{_HF_KINDS[kind]}{rest.replace('--', '/')}/resolve/"
        refs = _read_refs(repo_dir)
        blobs = os.path.join(repo_dir, "blobs")
        keys: dict[str, list[str]] = {}                       # blob name -> URLs
        loose: list[Entry] = []                               # snapshot files that are not links into blobs/
        snaps = os.path.join(repo_dir, "snapshots")
        for commit in sorted(os.listdir(snaps)) if os.path.isdir(snaps) else []:
            root = os.path.join(snaps, commit)
            revisions = [commit] + refs.get(commit, [])
            for dirpath, dirnames, filenames in os.walk(root):
                dirnames.sort()
                for f in sorted(filenames):
                    p = os.path.join(dirpath, f)
                    rel = os.path.relpath(p, root).replace(os.sep, "/")
                    urls = [base + quote(r, safe="") + "/" + quote(rel) for r in revisions]
                    target = os.path.realpath(p)
                    if os.path.islink(p) and os.path.dirname(target) == os.path.realpath(blobs):
                        keys.setdefault(os.path.basename(target), []).extend(urls)
                    else:
                        loose.append(Entry(p, None, urls))
        for name in sorted(os.listdir(blobs)) if os.path.isdir(blobs) else []:
            if _HEX64.fullmatch(name):
                expect = bytes.fromhex(name)                  # LFS: named by its SHA-256
            elif _HEX40.fullmatch(name):
                expect = None                                 # a regular git file, named by its git SHA-1
            else:
                continue                                      # *.incomplete and strays
            yield Entry(os.path.join(blobs, name), expect, keys.get(name, []))
        yield from loose


def import_entries(eng, entries, link: bool = False, page: int = 1024) -> dict:
    """Import entries through ``eng.import_files`` in pages of about `page` files.  Returns a summary: counts per
    status name, bytes imported, the entries that did not hash to their names, and the number of aliases entered."""
    from . import _lib
    names = {getattr(_lib, n): n for n in dir(_lib) if n.startswith("DM_E") or n == "DM_OK"}
    summary = {"status": {}, "bytes_imported": 0, "corrupt": [], "aliases": 0}
    batch: list[Entry] = []

    def flush():
        paths, expect, keys, owner = [], [], [], []
        for k, ent in enumerate(batch):
            for key in ent.keys or [None]:                    # one row per key: the engine imports a path once
                paths.append(ent.path)
                expect.append(ent.expect)
                keys.append(key)
                owner.append(k)
        res = eng.import_files(paths, expect=expect, keys=keys, link=link) if paths else []
        first: dict[int, tuple[int, bytes]] = {}
        for k, (st, dig), key in zip(owner, res, keys):
            first.setdefault(k, (st, dig))
            if st == DM_OK and key is not None:
                summary["aliases"] += 1
        for k, ent in enumerate(batch):
            st, dig = first[k]
            name = names.get(st, str(st))
            summary["status"][name] = summary["status"].get(name, 0) + 1
            if st == DM_OK:
                try:
                    summary["bytes_imported"] += os.path.getsize(ent.path)
                except OSError:
                    pass
            elif name == "DM_ECORRUPT":
                summary["corrupt"].append({"path": ent.path, "expected": ent.expect.hex(), "got": dig.hex()})
        batch.clear()

    for ent in entries:
        batch.append(ent)
        if len(batch) >= page:
            flush()
    flush()
    return summary
