#!/usr/bin/env python3
"""Regenerates tests/golden/*.json from sources that exist in THIS container.

Run from a checkout of the reference:  python tests/golden/make_golden.py <path to moeru-ai/demodel checkout>
(without the path only fips_vectors.json is rewritten)

1. reference_fixture.json — the only byte-level fixture the reference ships:
   the xxd dump of a cached, gzip-encoded Ollama manifest body at
   demodel/CONTRIBUTING.md:76-99, plus the manifest JSON it inflates
   to (CONTRIBUTING.md:128-153).  The reference states no digest for either;
   the digests recorded here are hashlib's (cross-checked against OpenSSL by
   tests/test_oracle.py).
2. fips_vectors.json — FIPS 180-4 / NIST CAVP known answers for SHA-256 (the
   published digests, typed in from the standard's examples, and re-verified
   against hashlib when this script runs).
"""
import gzip
import hashlib
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(sys.argv[1], "CONTRIBUTING.md") if len(sys.argv) > 1 else None


def reference_fixture():
    lines = open(REF, encoding="utf-8", errors="replace").read().split("\n")
    body = bytearray()
    for ln in lines[75:99]:                       # CONTRIBUTING.md:76-99
        m = re.match(r"^([0-9a-f]{8}): ((?:[0-9a-f]{2,4} ?)+) ", ln)
        assert m, ln
        assert int(m.group(1), 16) == len(body)
        body += bytes.fromhex(m.group(2).replace(" ", ""))
    raw = gzip.decompress(bytes(body))
    manifest = json.loads(raw)
    return {
        "source": "moeru-ai/demodel @ fb8342aa CONTRIBUTING.md:76-99 (xxd of .cache/1b8c2ef6c820e0c0)",
        "gzip_body_hex": bytes(body).hex(),
        "gzip_body_len": len(body),
        "gzip_body_sha256": hashlib.sha256(bytes(body)).hexdigest(),
        "inflated_len": len(raw),
        "inflated_sha256": hashlib.sha256(raw).hexdigest(),
        "inflated_utf8": raw.decode(),
        "manifest_layers": [
            {"mediaType": l["mediaType"], "digest": l["digest"], "size": l["size"]}
            for l in [manifest["config"]] + manifest["layers"]
        ],
        "digest_note": "digests computed with hashlib in the build container; the reference states none",
    }


FIPS = [
    # (name, message spec, published SHA-256)
    ("empty", {"ascii": ""}, "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"),
    ("abc", {"ascii": "abc"}, "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"),
    ("448bit", {"ascii": "abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq"},
     "248d6a61d20638b8e5c026930c3e6039a33ce45964ff2167f6ecedd419db06c1"),
    ("896bit", {"ascii": "abcdefghbcdefghicdefghijdefghijkefghijklfghijklmghijklmnhijklmnoijklmnopjklmnopq"
                         "klmnopqrlmnopqrsmnopqrstnopqrstu"},
     "cf5b16a778af8380036ce59e7b0492370b249b11e8f07a51afac45037afee9d1"),
    ("million_a", {"repeat": "a", "count": 1000000},
     "cdc76e5c9914fb9281a1c7e284d73e67f1809a48a497200e046d39ccc7112cd0"),
    # NIST CAVP SHA256ShortMsg.rsp samples
    ("cavp_len8", {"hex": "d3"}, "28969cdfa74a12c82f3bad960b0b000aca2ac329deea5c2328ebc6f2ba9802c1"),
    ("cavp_len16", {"hex": "11af"}, "5ca7133fa735326081558ac312c620eeca9970d1e70a4b95533d956f072d1f98"),
    ("cavp_len512", {"hex": "5a86b737eaea8ee976a0a24da63e7ed7eefad18a101c1211e2b3650c5187c2a8"
                            "a650547208251f6d4237e661c7bf4c77f335390394c37fa1a9f9be836ac28509"},
     "42e61e174fbb3897d6dd6cef3dd2802fe67b331953b06114a65c772859dfc1aa"),
]


def fips_vectors():
    out = []
    for name, spec, digest in FIPS:
        if "ascii" in spec:
            msg = spec["ascii"].encode()
        elif "hex" in spec:
            msg = bytes.fromhex(spec["hex"])
        else:
            msg = spec["repeat"].encode() * spec["count"]
        assert hashlib.sha256(msg).hexdigest() == digest, name
        out.append({"name": name, "message": spec, "sha256": digest})
    return out


def main():
    with open(os.path.join(HERE, "fips_vectors.json"), "w") as f:
        json.dump(fips_vectors(), f, indent=1)
    if REF and os.path.exists(REF):
        with open(os.path.join(HERE, "reference_fixture.json"), "w") as f:
            json.dump(reference_fixture(), f, indent=1)
    else:
        print("no reference checkout given: reference_fixture.json left as committed")


if __name__ == "__main__":
    main()
