"""Manifest-aware prefetch (SURVEY.md §8f-4), host-side mirror of
dm_manifest_parse / dm_manifest_prefetch.

An Ollama / OCI pull fetches the image manifest first (shape: the reference's
cached fixture, demodel/CONTRIBUTING.md:128-153); every layer's digest
and size is known from it, so the proxy can reserve and verify each layer
stream before its body arrives.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

from . import _lib
from ._lib import DmLayer, check


@dataclass(frozen=True)
class Layer:
    digest: bytes
    size: int
    media_type: str


def parse_manifest(body: bytes) -> list[Layer]:
    """Descriptors of a manifest body in document order (config first)."""
    lib = _lib.load()
    n = C.c_uint32()
    check(lib.dm_manifest_parse(body, len(body), None, 0, C.byref(n)), "dm_manifest_parse")
    arr = (DmLayer * max(n.value, 1))()
    check(lib.dm_manifest_parse(body, len(body), arr, n.value, C.byref(n)), "dm_manifest_parse")
    return [Layer(bytes(arr[i].digest), int(arr[i].size), arr[i].media_type.decode(errors="replace"))
            for i in range(n.value)]


def prefetch(engine, layers: list[Layer]) -> list[int]:
    """Pre-open one verified stream per layer not yet cached; 0 = already a hit."""
    lib = _lib.load()
    n = len(layers)
    arr = (DmLayer * max(n, 1))()
    for i, l in enumerate(layers):
        arr[i].digest[:] = l.digest
        arr[i].size = l.size
        arr[i].media_type = l.media_type.encode()[:95]
    ids = (C.c_uint64 * max(n, 1))()
    check(lib.dm_manifest_prefetch(engine._h, arr, n, ids), "dm_manifest_prefetch")
    return [int(ids[i]) for i in range(n)]
