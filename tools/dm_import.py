#!/usr/bin/env python3
"""Import a host's existing model files into a demodel cache directory, each hashed on the GPU (dm_cache_import).

  dm_import.py --cas-dir D --ollama ~/.ollama/models        an Ollama models directory
  dm_import.py --cas-dir D --hf-cache ~/.cache/huggingface/hub

Run it at deployment over the node's model caches, or after copying another node's cache over, before the proxy
starts on D (or with the proxy's engine stopped).  --link hard-links files into D where D is on the same filesystem
instead of copying them.  The source directory is only read.  Prints one JSON line: counts per status, bytes imported,
the files that did not hash to the digest their name gives, and the number of aliases entered.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import demodel_b200  # noqa: E402
from demodel_b200 import importer  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cas-dir", required=True)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--ollama", metavar="DIR")
    src.add_argument("--hf-cache", metavar="DIR")
    ap.add_argument("--link", action="store_true")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--hbm-cas-bytes", type=int, default=256 << 20, help="the engine's HBM arena (the import uses none)")
    args = ap.parse_args(argv)
    entries = importer.ollama_entries(args.ollama) if args.ollama else importer.hf_entries(args.hf_cache)
    with demodel_b200.Engine(device=args.device, hbm_cas_bytes=args.hbm_cas_bytes, cas_dir=args.cas_dir) as eng:
        summary = importer.import_entries(eng, entries, link=args.link)
    summary["source"] = args.ollama or args.hf_cache
    print(json.dumps(summary))
    return 0 if not summary["corrupt"] else 1


if __name__ == "__main__":
    sys.exit(main())
