#!/usr/bin/env python3
"""Cycles per iteration that ptxas itself scheduled: sum of the stall counts in the SASS control words.

For a single in-order warp running fixed-latency integer code (the deep / group kernels' serial phase) the
issue time of the loop is, to first order, the sum over its instructions of the `stall` field ptxas encoded
(bits 105..108 of each 128-bit instruction: cycles to wait before issuing the next one) - ncu shows exactly
that for the shipped kernel: `selected` 1.00 + `wait` 1.02 per issue and nothing else
(ncu metrics of the deep kernel).  Comparing this number with the measured launch time says whether
a form is limited by ptxas' own schedule or by something the hardware adds on top.

  cuobjdump -sass build/sha256_kernels.o > all.sass; tools/sass_stalls.py all.sass 'deep_kernelILi7E'
"""
import collections
import re
import sys


def parse(path, func):
    lines = open(path).read().split("\n")
    cur, rows, i = None, [], 0
    while i < len(lines):
        m = re.search(r"Function : (\S+)", lines[i])
        if m:
            cur = m.group(1)
        if cur and func in cur:
            m = re.match(r"\s*/\*([0-9a-f]{4,5})\*/\s+(.*?)\s*;\s*/\* (0x[0-9a-f]+) \*/", lines[i])
            if m and i + 1 < len(lines):
                m2 = re.search(r"/\* (0x[0-9a-f]+) \*/", lines[i + 1])
                if m2:
                    ctrl = int(m2.group(1), 16) >> 41
                    text = re.sub(r"^@!?U?P\w+\s+", "", m.group(2).strip())
                    rows.append({"addr": int(m.group(1), 16), "text": text, "op": text.split()[0].split(".")[0],
                                 "stall": ctrl & 0xf, "yield": (ctrl >> 4) & 1, "wbar": (ctrl >> 5) & 7,
                                 "rbar": (ctrl >> 8) & 7, "wait": (ctrl >> 11) & 0x3f})
                    i += 1
        i += 1
    return rows


def main():
    rows = parse(sys.argv[1], sys.argv[2])
    lds = [k for k, r in enumerate(rows) if r["op"] == "LDS"]
    if len(lds) < 2:
        sys.exit("no LDS-delimited loop found in " + sys.argv[2])
    loop = rows[lds[0]:lds[-1] + 1]
    # the phase-2 loop body runs from its first LDS to the backward branch: extend to the closing BRA
    end = lds[-1]
    while end + 1 < len(rows) and rows[end]["op"] != "BRA":
        end += 1
    loop = rows[lds[0]:end + 1]
    ops = collections.Counter(r["op"] for r in loop)
    total = sum(max(r["stall"], 1) for r in loop)
    rounds = max(16, 16 * round(ops["SHF"] / 96))     # 6 rotations per round (+ a few address shifts): 64 (unrolled) or 16 (rolled) rounds per iteration
    print(f"{sys.argv[2]}: {len(loop)} instructions in the loop ({rounds} rounds per iteration): " + ", ".join(f"{k} {v}" for k, v in ops.most_common(8)))
    print(f"  sum of ptxas stall counts = {total} cycles per iteration = {total / rounds:.2f} cycles per round"
          f" -> {1.98e9 / (total / rounds) / 1e6:.1f} MB/s per stream at 1.98 GHz (phase 2 only)")


if __name__ == "__main__":
    main()
