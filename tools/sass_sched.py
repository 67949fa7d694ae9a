#!/usr/bin/env python3
"""Static issue-timing estimate for a straight-line SASS loop run by ONE warp.

For the single-warp serial phase of sha256_warp_kernel (one warp per stream, alone on
its sub-partition) nothing hides latency, so the cycles per round can be estimated
from the SASS alone.  Model (pipe rates and latencies as tools/ubench/pipemix.cu and
chainlat.cu measure them):

  * in-order issue, at most one instruction per cycle;
  * the ALU pipe (SHF, LOP3, IADD3, PRMT, VIADD, ISETP, MOV ...) and the FMA pipe
    (IMAD*) each accept one warp-instruction per 2 cycles and run concurrently;
  * fixed latency 4 cycles to a consumer on the same pipe, 5 across pipes;
  * LDS: 29 cycles to its consumer (scoreboard), LSU pipe, 2-cycle issue.

Usage:
  cuobjdump -sass build/sha256_kernels.o > all.sass
  tools/sass_sched.py all.sass 'warp_kernelILi0ELi1ELb0EE' [--iters 3]   # <form 0, S = 1, one warp>

Picks the loop between the first and last LDS of the named function (the phase-2
block loop), replays it `iters` times and prints cycles per iteration in steady
state, the pipe-issue lower bounds and the critical-path bound.  It is a ranking
tool for candidate round orderings when no GPU is at hand.  On an H100 SXM the
model reads 35.0 cycles per round for form 0 and 24.3 for form 7 at S = 1; measured at
1.98 GHz (256 x 1 MiB per launch) they take 37.8 and 26.5.
"""
import argparse
import re
import sys

ALU = {"SHF", "LOP3", "IADD3", "PRMT", "VIADD", "ISETP", "MOV", "SEL", "LEA", "IABS", "IMNMX", "VIMNMX", "PLOP3",
       "UMOV", "UIADD3", "ULOP3", "USHF", "UISETP", "ULEA", "R2UR", "S2UR", "NOP", "CS2R"}
FMA = {"IMAD"}
LSU = {"LDS", "STS", "LDG", "STG", "LD", "ST", "LDC", "LDCU"}


def parse(path, func):
    cur = None
    rows = []
    for line in open(path):
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur is None or func not in cur:
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,5})\*/\s+(.*?);", line)
        if not m:
            continue
        text = m.group(2).strip()
        pred = None
        pm = re.match(r"(@!?U?P\d|@!?PT)\s+(.*)", text)
        if pm:
            pred, text = pm.group(1), pm.group(2)
        op, _, rest = text.partition(" ")
        base = op.split(".")[0]
        ops = [o.strip() for o in rest.split(",")] if rest else []
        rows.append((int(m.group(1), 16), op, base, ops, pred))
    return rows


def regs_of(tok):
    return [int(x) for x in re.findall(r"(?<![A-Za-z])R(\d+)", tok)]


def decode(row):
    _, op, base, ops, _ = row
    width = 4 if ".128" in op else 2 if (".64" in op or ".WIDE" in op) else 1
    dst, src = [], []
    if base in ("STS", "STG", "ST", "BRA", "BAR", "EXIT", "NOP", "WARPSYNC", "BSSY", "BSYNC"):
        for o in ops:
            src += regs_of(o)
        if base in ("STS", "STG", "ST") and len(ops) >= 2:
            r = regs_of(ops[-1])
            if r:
                src += [r[0] + i for i in range(width)]
    else:
        if ops:
            d = regs_of(ops[0])
            if d and not ops[0].startswith("["):
                dst = [d[0] + i for i in range(width)]
            elif ops[0].startswith("P") or ops[0].startswith("UP"):
                dst = []
        for o in ops[1:]:
            src += regs_of(o)
    pipe = "alu" if base in ALU else "fma" if base in FMA else "lsu" if base in LSU else "other"
    return dst, src, pipe


WIDE_RT, WIDE_LAT = 2, 4      # IMAD.WIDE / IMAD.HI issue interval and latency: unmeasured, set by --wide-rt / --wide-lat


def simulate(body, iters):
    ready = {}            # reg -> (cycle the value is available to a same-pipe consumer, producing pipe)
    pipe_free = {"alu": 0, "fma": 0, "lsu": 0, "other": 0}
    t = 0
    marks = []
    crit = {}
    for it in range(iters):
        for row in body:
            dst, src, pipe = decode(row)
            start = max(t, pipe_free[pipe])
            for r in src:
                if r in ready:
                    avail, ppipe, lat = ready[r]
                    a = avail + (0 if (ppipe == pipe or lat >= 29) else 1)
                    start = max(start, a)
            wide = row[2] == "IMAD" and (".WIDE" in row[1] or ".HI" in row[1])
            lat = 29 if row[2] in ("LDS", "LDG", "LDC") else WIDE_LAT if wide else 4
            for r in dst:
                ready[r] = (start + lat, pipe, lat)
            pipe_free[pipe] = start + (WIDE_RT if wide else 2)
            t = start + 1
        marks.append(t)
    return marks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("sass")
    ap.add_argument("func")
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=64, help="rounds per loop iteration")
    ap.add_argument("--wide-rt", type=int, default=2, help="assumed issue interval of IMAD.WIDE / IMAD.HI")
    ap.add_argument("--wide-lat", type=int, default=4, help="assumed latency of IMAD.WIDE / IMAD.HI")
    a = ap.parse_args()
    global WIDE_RT, WIDE_LAT
    WIDE_RT, WIDE_LAT = a.wide_rt, a.wide_lat
    rows = parse(a.sass, a.func)
    if not rows:
        sys.exit("function not found")
    lds = [i for i, r in enumerate(rows) if r[2] == "LDS"]
    if not lds:
        sys.exit("no LDS in function")
    first = lds[0]
    end = next(i for i in range(lds[-1], len(rows)) if rows[i][2] == "BRA")
    # the loop head is the branch target; fall back to the first LDS
    m = re.search(r"0x([0-9a-f]+)", " ".join(rows[end][3]))
    if m:
        tgt = int(m.group(1), 16)
        idx = [i for i, r in enumerate(rows) if r[0] == tgt]
        if idx and idx[0] <= first:
            first = idx[0]
    body = rows[first:end + 1]
    n = {"alu": 0, "fma": 0, "lsu": 0, "other": 0}
    for r in body:
        n[decode(r)[2]] += 1
    marks = simulate(body, a.iters)
    per = marks[-1] - marks[-2]
    print(f"{a.func}: loop of {len(body)} instructions  alu={n['alu']} fma={n['fma']} lsu={n['lsu']} other={n['other']}")
    print(f"  issue bounds per iteration: alu {2 * n['alu']}  fma {2 * n['fma']}  total {len(body)}")
    print(f"  simulated: {per} cycles per iteration = {per / a.rounds:.2f} cycles per round "
          f"-> {1.9e9 / (per / a.rounds) / 1e6:.0f} MB/s per stream at 1.9 GHz (phase 2 only)")


if __name__ == "__main__":
    main()
