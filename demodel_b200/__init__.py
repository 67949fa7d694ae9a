"""demodel_b200 — H100-native blob hash-and-cache engine (host-side mirror).

The product is ``libdemodel_b200.so`` (hand-written sm_90a SHA-256 kernels +
the ingest/CAS engine behind the C-ABI in ``include/demodel_b200.h``).  The
Python here is a thin ctypes mirror for tests and the benchmark; it never
computes a digest itself and it fails loudly when the library is missing.
"""
from ._lib import (DM_ECORRUPT, DM_ECUDA, DM_EINVAL, DM_EIO, DM_ENODEV, DM_ENOENT, DM_ENOMEM, DM_ERANGE, DM_ESTATE,
                   DM_OK, DmError, LIB_PATH, load)
from .engine import Engine, shard_of, synth_fill_host
from .shard import ShardRouter

__all__ = ["Engine", "ShardRouter", "shard_of", "synth_fill_host", "DmError", "load", "LIB_PATH",
           "DM_OK", "DM_EINVAL", "DM_ENOMEM", "DM_ENOENT", "DM_ECUDA", "DM_ESTATE", "DM_EIO", "DM_ENODEV", "DM_ERANGE",
           "DM_ECORRUPT"]
