"""ctypes binding of include/demodel_b200.h.

The product is the C-ABI shared library ``libdemodel_b200.so`` (CUDA kernels +
engine).  This module only declares its signatures.  There is no fallback: if
the library is missing, loading raises and every op fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdemodel_b200.so")

DM_OK, DM_EINVAL, DM_ENOMEM, DM_ENOENT, DM_ECUDA, DM_ESTATE, DM_EIO, DM_ENODEV, DM_ERANGE, DM_ECORRUPT = (
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9)

DM_F_NO_HBM_CAS = 0x1
DM_F_DISK_SYNC = 0x2
DM_F_NUMA_LOCAL = 0x4
DM_F_DISK_DIRECT = 0x8
DM_ING_HASH_ONLY = 0x1
DM_ING_REPLACE = 0x2
DM_ING_FORCE_WIDE = 0x4
DM_ING_FORCE_DEEP = 0x8
DM_IMP_LINK = 0x1
DM_RM_ALIASES = 0x1
DM_RM_PARTIAL = 0x2


class DmConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("device", C.c_int32),
        ("hbm_cas_bytes", C.c_uint64),
        ("ring_bytes", C.c_uint64),
        ("slab_bytes", C.c_uint32),
        ("max_streams", C.c_uint32),
        ("cas_dir", C.c_char_p),
        ("flags", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class DmStats(C.Structure):
    _fields_ = [
        ("bytes_ingested", C.c_uint64),
        ("bytes_hashed", C.c_uint64),
        ("bytes_served", C.c_uint64),
        ("blobs_committed", C.c_uint64),
        ("blobs_mismatched", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("launches_wide", C.c_uint64),
        ("launches_deep", C.c_uint64),
        ("kernel_ms", C.c_double),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("hbm_cas_used", C.c_uint64),
        ("hbm_cas_capacity", C.c_uint64),
        ("open_streams", C.c_uint64),
        ("ring_waits", C.c_uint64),
        ("launches_group", C.c_uint64),
        ("ring_slabs_total", C.c_uint64),
        ("ring_slabs_free", C.c_uint64),
        ("open_readers", C.c_uint64),
        ("free_stream_slots", C.c_uint64),
        ("numa_node", C.c_int64),
        ("aliases", C.c_uint64),
        ("suspended", C.c_uint64),
        ("packed_bodies", C.c_uint64),
        ("packs", C.c_uint64),
    ]


class DmLayer(C.Structure):
    _fields_ = [("digest", C.c_uint8 * 32), ("size", C.c_uint64), ("media_type", C.c_char * 96)]


class DmDiskUsage(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("reserved", C.c_uint32),
        ("limit_bytes", C.c_uint64),
        ("used_bytes", C.c_uint64),
        ("blob_files", C.c_uint64),
        ("blob_bytes", C.c_uint64),
        ("staging_bytes", C.c_uint64),
        ("partial_bytes", C.c_uint64),
        ("evicted_files", C.c_uint64),
        ("evicted_bytes", C.c_uint64),
        ("refused", C.c_uint64),
    ]


class DmCheckpoint(C.Structure):
    _fields_ = [("h", C.c_uint32 * 8), ("bytes", C.c_uint64), ("abi", C.c_uint32), ("reserved", C.c_uint32)]


# name -> (restype, argtypes); every symbol include/demodel_b200.h declares.
_P = C.c_void_p
_U8P = C.POINTER(C.c_uint8)
_U64P = C.POINTER(C.c_uint64)
SIGNATURES = {
    "dm_abi_version": (C.c_uint32, []),
    "dm_device_count": (C.c_int, []),
    "dm_engine_create": (C.c_int, [C.POINTER(DmConfig), C.POINTER(_P)]),
    "dm_engine_destroy": (None, [_P]),
    "dm_engine_stats": (C.c_int, [_P, C.POINTER(DmStats)]),
    "dm_strerror": (C.c_char_p, [C.c_int]),
    "dm_last_error": (C.c_char_p, []),
    "dm_error_detail": (C.c_int, [_P, C.c_uint64, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dm_shard_of": (C.c_uint32, [_P, C.c_uint32]),
    "dm_streams_per_warp": (C.c_uint32, [C.c_uint32]),
    "dm_default_kernel_variant": (C.c_uint32, [C.c_int]),
    "dm_stream_open": (C.c_int, [_P, _P, C.c_uint64, _U64P]),
    "dm_stream_write": (C.c_int, [_P, C.c_uint64, _P, C.c_size_t]),
    "dm_stream_write_at": (C.c_int, [_P, C.c_uint64, C.c_uint64, _P, C.c_size_t]),
    "dm_stream_checkpoint": (C.c_int, [_P, C.c_uint64, C.POINTER(DmCheckpoint)]),
    "dm_stream_resume": (C.c_int, [_P, C.POINTER(DmCheckpoint), _P, C.c_uint64, _U64P]),
    "dm_stream_set_meta": (C.c_int, [_P, C.c_uint64, C.c_char_p, C.c_char_p]),
    "dm_stream_acquire": (C.c_int, [_P, C.c_uint64, C.POINTER(_P), C.POINTER(C.c_size_t)]),
    "dm_stream_commit": (C.c_int, [_P, C.c_uint64, C.c_size_t]),
    "dm_stream_flush": (C.c_int, [_P, C.c_uint64]),
    "dm_stream_finish": (C.c_int, [_P, C.c_uint64, _P, C.POINTER(C.c_int)]),
    "dm_stream_abort": (C.c_int, [_P, C.c_uint64]),
    "dm_cache_contains": (C.c_int, [_P, _P, _U64P]),
    "dm_cache_open": (C.c_int, [_P, _P, _U64P, _U64P]),
    "dm_cache_open_verified": (C.c_int, [_P, _P, _U64P, _U64P]),
    "dm_cache_open_verified_ring": (C.c_int, [_P, _P, _U64P, _U64P]),
    "dm_cache_open_verified_range": (C.c_int, [_P, _P, C.c_uint64, C.c_uint64, _U64P, _U64P]),
    "dm_cache_read": (C.c_int, [_P, C.c_uint64, C.c_uint64, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dm_cache_meta": (C.c_int, [_P, C.c_uint64, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dm_cache_close": (C.c_int, [_P, C.c_uint64]),
    "dm_cache_evict": (C.c_int, [_P, _P]),
    "dm_cache_remove": (C.c_int, [_P, _P, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32)]),
    "dm_cache_promote": (C.c_int, [_P, _P, C.c_uint32, C.POINTER(C.c_int32)]),
    "dm_cache_verify": (C.c_int, [_P, _P, C.c_uint32, C.POINTER(C.c_int32)]),
    "dm_cache_list": (C.c_int, [_P, _P, _P, _U64P, C.c_uint32, C.POINTER(C.c_uint32)]),
    "dm_cache_import": (C.c_int, [_P, C.POINTER(C.c_char_p), _P, C.POINTER(C.c_char_p), C.c_uint32, C.c_uint32, _P,
                                  C.POINTER(C.c_int32)]),
    "dm_cache_export": (C.c_int, [_P, _P, C.POINTER(C.c_char_p), C.c_uint32, C.POINTER(C.c_int32)]),
    "dm_cache_set_disk_limit": (C.c_int, [_P, C.c_uint64]),
    "dm_cache_disk_usage": (C.c_int, [_P, C.POINTER(DmDiskUsage)]),
    "dm_cache_follow": (C.c_int, [_P, _P, _U64P, _U64P]),
    "dm_cache_alias_put": (C.c_int, [_P, C.c_char_p, _P]),
    "dm_cache_alias_get": (C.c_int, [_P, C.c_char_p, _P]),
    "dm_cache_alias_del": (C.c_int, [_P, C.c_char_p]),
    "dm_cache_alias_list": (C.c_int, [_P, C.c_char_p, C.c_char_p, _P, C.c_size_t, _P, C.c_uint32,
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_int)]),
    "dm_stream_suspend": (C.c_int, [_P, C.c_uint64, _U64P]),
    "dm_stream_resume_saved": (C.c_int, [_P, _P, C.c_uint64, _U64P, _U64P]),
    "dm_gunzip": (C.c_int, [_P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dm_cache_device_extents": (C.c_int, [_P, C.c_uint64, C.POINTER(_P), _U64P, C.c_uint32]),
    "dm_ingest_device": (C.c_int, [_P, _P, _U64P, _U64P, C.c_uint32, _P, _P, _P, C.c_uint32, C.POINTER(C.c_double)]),
    "dm_manifest_parse": (C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(DmLayer), C.c_uint32, C.POINTER(C.c_uint32)]),
    "dm_manifest_prefetch": (C.c_int, [_P, C.POINTER(DmLayer), C.c_uint32, _U64P]),
    "dm_synth_fill_host": (None, [C.c_uint64, C.c_uint64, C.c_uint64, _P, C.c_size_t]),
    "dm_synth_fill_device": (C.c_int, [_P, C.c_uint64, C.c_uint64, C.c_uint64, _P, C.c_size_t]),
    "dm_synth_fill_device_many": (C.c_int, [_P, C.c_uint64, C.c_uint64, _P, _U64P, _U64P, C.c_uint32]),
    "dm_proxy_drive": (C.c_int, [_P, _P, _U64P, C.c_uint32, _P, C.c_size_t, C.c_uint32, C.c_int, C.c_int,
                                 _P, _P, C.POINTER(C.c_double)]),
    "dm_proxy_fetch": (C.c_int, [_P, C.c_char_p, _P, C.c_uint64, _P, C.c_size_t, _P, C.POINTER(C.c_int)]),
    "dm_proxy_request": (C.c_int, [_P, C.c_char_p, _U64P, _U64P]),
    "dm_proxy_manifest": (C.c_int, [_P, _P, C.c_uint64, C.c_char_p, C.c_size_t, C.POINTER(DmLayer), _U64P, C.c_uint32,
                                    C.POINTER(C.c_uint32)]),
    "dm_proxy_serve": (C.c_int, [_P, _P, C.c_uint32, _P, _U64P, C.c_size_t, C.c_int, C.POINTER(C.c_double)]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen the engine and bind every declared symbol.  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C demodel_b200/csrc`.  There is no CPU fallback for the hash path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class DmError(RuntimeError):
    def __init__(self, code: int, where: str):
        lib = load()
        detail = lib.dm_last_error().decode(errors="replace")
        msg = lib.dm_strerror(code).decode()
        super().__init__(f"{where}: {msg} ({code})" + (f": {detail}" if detail else ""))
        self.code = code


def check(code: int, where: str) -> int:
    if code != DM_OK:
        raise DmError(code, where)
    return code
