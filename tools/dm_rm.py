#!/usr/bin/env python3
"""Remove models from a demodel cache directory (dm_cache_remove, dm_cache_alias_del).

  dm_rm.py --cas-dir D --digest HEX [HEX ...]                    these blobs and every alias naming them
  dm_rm.py --cas-dir D --alias-prefix P                          the aliases under P, and the blobs only they name
  dm_rm.py --cas-dir D --hf-repo ORG/NAME [--revision R]         a HuggingFace repository's resolve/ URLs (one revision)
  dm_rm.py --cas-dir D --ollama MANIFEST_URL                     an Ollama / OCI model: its manifest and its layers

Aliases are removed as selected.  A blob is removed only when no alias outside the removed set still names it, so the
same tokenizer.json in two repositories survives the removal of one of them.  For --ollama, a layer stays while
another aliased manifest lists it (a licence, params or base weights shared by two models).  Run it with the proxy's
engine on D stopped, as dm_import.py.  --dry-run prints the plan and removes nothing.  Prints one JSON line: the
aliases and blobs removed, the blobs kept because something else names them, the bytes freed and the status of each
blob that was not removed.
"""
import argparse
import json
import os
import sys
from urllib.parse import quote

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import demodel_b200  # noqa: E402
from demodel_b200 import _lib, importer  # noqa: E402
from demodel_b200.manifest import parse_manifest  # noqa: E402


def _manifest_layers(eng, digest):
    """Digests a cached manifest lists (config and layers); empty when it is not cached or not a manifest."""
    body = eng.fetch(digest)
    if body is None:
        return set()
    try:
        return {layer.digest for layer in parse_manifest(body)}
    except demodel_b200.DmError:
        return set()


def plan(eng, args):
    """(aliases to delete, digests to remove, digests kept because an alias outside the set names them)."""
    aliases = dict(eng.alias_list(""))
    if args.digest:
        digests = {bytes.fromhex(h) for h in args.digest}
        return sorted(k for k, d in aliases.items() if d in digests), digests, set()
    if args.ollama:
        top = aliases.get(args.ollama)
        if top is None:
            raise SystemExit(f"no alias {args.ollama!r} in this cache")
        dead = [args.ollama]
        wanted = {top} | _manifest_layers(eng, top)
        keep = set()
        for key, d in aliases.items():                    # every other aliased manifest keeps what it lists
            if key != args.ollama and "/manifests/" in key:
                keep |= {d} | _manifest_layers(eng, d)
    else:
        if args.hf_repo:
            prefix = f"{importer.HF_ENDPOINT}/{args.hf_repo}/resolve/"
            if args.revision:
                prefix += quote(args.revision, safe="") + "/"
        else:
            prefix = args.alias_prefix
        dead = [k for k in aliases if k.startswith(prefix)]
        wanted = {aliases[k] for k in dead}
        keep = set()
    dead_set = set(dead)
    keep |= {d for k, d in aliases.items() if k not in dead_set}
    return sorted(dead), wanted - keep, wanted & keep


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cas-dir", required=True)
    what = ap.add_mutually_exclusive_group(required=True)
    what.add_argument("--digest", nargs="+", metavar="HEX")
    what.add_argument("--alias-prefix", metavar="P")
    what.add_argument("--hf-repo", metavar="ORG/NAME")
    what.add_argument("--ollama", metavar="MANIFEST_URL")
    ap.add_argument("--revision", help="with --hf-repo: only the resolve/ URLs of this revision (a commit or a ref)")
    ap.add_argument("--dry-run", action="store_true")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--hbm-cas-bytes", type=int, default=256 << 20, help="the engine's HBM arena (removal uses none)")
    args = ap.parse_args(argv)
    if args.revision and not args.hf_repo:
        ap.error("--revision needs --hf-repo")
    if args.digest and any(len(h) != 64 for h in args.digest):
        ap.error("a digest is 64 hex digits")
    names = {getattr(_lib, n): n for n in dir(_lib) if n.startswith("DM_E") or n == "DM_OK"}
    with demodel_b200.Engine(device=args.device, hbm_cas_bytes=args.hbm_cas_bytes, cas_dir=args.cas_dir) as eng:
        dead, blobs, kept = plan(eng, args)
        blobs = sorted(blobs)
        sizes = {d: eng.cache_contains(d) or 0 for d in blobs}
        out = {"dry_run": args.dry_run, "aliases_removed": dead, "kept": sorted(d.hex() for d in kept)}
        if args.dry_run:
            out.update(removed=[d.hex() for d in blobs if sizes[d]], bytes_freed=sum(sizes.values()), not_removed={})
        else:
            for key in dead:
                eng.alias_del(key)
            status = eng.cache_remove(blobs, partial=bool(args.digest))
            out["removed"] = [d.hex() for d, st in zip(blobs, status) if st == _lib.DM_OK]
            out["bytes_freed"] = sum(sizes[d] for d, st in zip(blobs, status) if st == _lib.DM_OK)
            out["not_removed"] = {d.hex(): names.get(st, str(st)) for d, st in zip(blobs, status) if st != _lib.DM_OK}
    print(json.dumps(out))
    return 0 if not any(v != "DM_ENOENT" for v in out["not_removed"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
