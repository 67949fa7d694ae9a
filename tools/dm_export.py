#!/usr/bin/env python3
"""Export the models a demodel cache directory holds, each file hashed on the GPU on its way out (dm_cache_export).

  dm_export.py --cas-dir D --ollama DIR          as an Ollama models directory (ollama run works there)
  dm_export.py --cas-dir D --hf-cache DIR        as a HuggingFace hub cache (HF_HUB_OFFLINE=1 works there)
  ... --only library/llama3:8b --only org/name   only these models / repositories

The names come from D's alias index (what dm_import.py and the proxy's body tee entered).  Run it with the proxy's
engine stopped, or on a copy of D.  D itself is only read.  The output directory can be carried to another machine and
used there directly, or imported into another cache with dm_import.py.  Prints one JSON line: counts per status, bytes
exported, the blobs whose copy did not hash to its name (run dm_cache_verify on D), and what was skipped and why.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import demodel_b200  # noqa: E402
from demodel_b200 import exporter  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cas-dir", required=True)
    dst = ap.add_mutually_exclusive_group(required=True)
    dst.add_argument("--ollama", metavar="DIR")
    dst.add_argument("--hf-cache", metavar="DIR")
    ap.add_argument("--only", action="append", metavar="NAME", help="a model (Ollama) or repository id (HuggingFace)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--hbm-cas-bytes", type=int, default=256 << 20, help="the engine's HBM arena (the export uses none)")
    args = ap.parse_args(argv)
    with demodel_b200.Engine(device=args.device, hbm_cas_bytes=args.hbm_cas_bytes, cas_dir=args.cas_dir) as eng:
        if args.ollama:
            plan = exporter.ollama_plan(eng, args.ollama, only=args.only)
        else:
            plan = exporter.hf_plan(eng, args.hf_cache, only=args.only)
        summary = exporter.export_entries(eng, plan)
    summary["destination"] = args.ollama or args.hf_cache
    print(json.dumps(summary))
    return 0 if not summary["corrupt"] else 1


if __name__ == "__main__":
    sys.exit(main())
