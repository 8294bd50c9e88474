#!/usr/bin/env python
"""sass_express.py -- SASS instructions per 4 KB unit of the express lane (scan_sum_express_kernel), read from the compiled object.

    python tools/sass_express.py [skywalking-banyandb_b200/build/scan_kernels.cu.o]

The object is built with -lineinfo (the Makefile's default), so `nvdisasm -g` tags every instruction with the source line it came
from; the innermost (inlined) line decides where it is counted.  The two-class copy of the unit decode is straight-line code, so
its static count is what a warp issues per unit:

    interior unit = the two-class copy (32 x swar_word2, loads, swar_begin / swar_end, vote: express_half, express_unit)
                    + the unit loop's own lines (neighbour words, packed scan, 64-bit multiply-add, ring wait and refill)
    edge unit     = interior unit + express_zero_edges (a unit that holds the body's first or last byte)

The three-class copy (the redo after a raised flag) and the general refill path (`issue`) are reported apart.  The script also
lists local-memory instructions (LDL / STL) in the two-class copy and on the unit loop's lines.

For comparison, the 2 KB chunk loop this replaced took about 512 instructions per interior chunk (256 per KB) and 644 per
masked edge chunk, about 4,360 per 15.8 KB bench page.
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "skywalking-banyandb_b200", "csrc")
KERNEL = "_ZN4bydb23scan_sum_express_kernelENS_10ScanParamsE"
UNIT_BYTES = 4096


def fn_lines(path, start_pat, end_pat=None):
    """[first, last] source lines of the function that starts at the first line matching start_pat (to its closing brace at
    column 0, or to the line before end_pat)."""
    lines = open(path).read().splitlines()
    a = next(i for i, t in enumerate(lines) if re.search(start_pat, t))
    if end_pat is not None:
        b = next(i for i in range(a + 1, len(lines)) if re.search(end_pat, lines[i])) - 1
    else:
        b = next(i for i in range(a + 1, len(lines)) if lines[i].startswith("}"))
    return a + 1, b + 1


def disassemble(obj):
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=d, stdout=subprocess.DEVNULL)
        cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
        if len(cubins) != 1:
            sys.exit(f"expected one cubin in {obj}, found {cubins}")
        return subprocess.check_output(["nvdisasm", "-g", "-c", os.path.join(d, cubins[0])], text=True)


def kernel_instructions(text):
    """[(address, source file basename, line, instruction text)] of the express kernel."""
    out, inside, where = [], False, None
    for line in text.splitlines():
        if re.match(r"\s*\.section\s", line):
            inside = f".text.{KERNEL}," in line
            continue
        if not inside:
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', line)
        if m:
            where = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and where:
            out.append((int(m.group(1), 16), where[0], where[1], m.group(2)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("obj", nargs="?", default=os.path.join(ROOT, "skywalking-banyandb_b200", "build", "scan_kernels.cu.o"))
    args = ap.parse_args()
    ins = kernel_instructions(disassemble(args.obj))
    if not ins:
        sys.exit("no express kernel with line info in " + args.obj)
    sk, ld = os.path.join(CSRC, "scan_kernels.cu"), os.path.join(CSRC, "lane_decode.cuh")
    regions = {
        "swar_word2": (ld, fn_lines(ld, r"void swar_word2\(")),
        "swar_word": (ld, fn_lines(ld, r"void swar_word\(")),
        "swar_begin/end": (ld, None),
        "express_zero_edges": (sk, fn_lines(sk, r"void express_zero_edges\(")),
        "keep_bytes": (sk, fn_lines(sk, r"void keep_bytes\(")),
        "express_half": (sk, fn_lines(sk, r"void express_half\(")),
        "express_unit": (sk, fn_lines(sk, r"ExpressUnit express_unit\(")),
        "ring_wait": (sk, fn_lines(sk, r"uint8_t \*ring_wait\(ExpressSmem")),
        "ring_fill": (sk, fn_lines(sk, r"void ring_fill\(")),
        "issue (general refill)": (sk, fn_lines(sk, r"auto issue = \[&\]", r"^\s+\};")),
        "unit loop": (sk, fn_lines(sk, r"for \(uint32_t j = 0; j < nst_k; \+\+j\)", r"last_byte = __shfl_sync\(0xffffffffu, last_byte, 0\);")),
    }
    b0 = fn_lines(ld, r"void swar_begin\(")
    e0 = fn_lines(ld, r"uint32_t swar_end\(")

    def region_of(f, line):
        if f == "lane_decode.cuh" and (b0[0] <= line <= b0[1] or e0[0] <= line <= e0[1]):
            return "swar_begin/end"
        for name, (path, span) in regions.items():
            if span and os.path.basename(path) == f and span[0] <= line <= span[1] and name != "unit loop":
                return name
        path, span = regions["unit loop"]
        if f == os.path.basename(path) and span[0] <= line <= span[1]:
            return "unit loop"
        return "elsewhere"

    tagged = [(a, region_of(f, l), t) for a, f, l, t in ins]
    # the two- and three-class copies: the address spans of their words, widened to the helper code around them
    w2 = [a for a, r, _ in tagged if r == "swar_word2"]
    w3 = [a for a, r, _ in tagged if r == "swar_word"]
    helpers = ("express_half", "express_unit", "swar_begin/end")

    def span(words, other):
        lo, hi = min(words), max(words)
        # extend over the helper instructions next to the copy (loads before the first word, vote / end after the last),
        # stopping at the other copy's words
        addrs = [a for a, r, _ in tagged]
        i, j = addrs.index(lo), addrs.index(hi)
        while i > 0 and tagged[i - 1][1] in helpers and tagged[i - 1][0] not in other:
            i -= 1
        while j + 1 < len(tagged) and tagged[j + 1][1] in helpers and tagged[j + 1][0] not in other:
            j += 1
        return tagged[i][0], tagged[j][0]

    s2, s3 = span(w2, set(w3)), span(w3, set(w2)) if w3 else (None, None)
    c2 = collections.Counter(r for a, r, _ in tagged if s2[0] <= a <= s2[1])
    c3 = collections.Counter(r for a, r, _ in tagged if s3[0] is not None and s3[0] <= a <= s3[1])
    loop_own = collections.Counter(r for a, r, _ in tagged if not (s2[0] <= a <= s2[1]) and not (s3[0] is not None and s3[0] <= a <= s3[1]))
    copy2 = sum(c2.values())
    scaffold = loop_own["unit loop"] + loop_own["ring_wait"] + loop_own["ring_fill"]
    interior = copy2 + scaffold
    zero = loop_own["express_zero_edges"] + loop_own["keep_bytes"]
    edge = interior + zero
    words = sum(c for r, c in c2.items() if r not in helpers)
    print(f"express kernel: {len(ins)} SASS instructions")
    print(f"two-class copy: {copy2} instructions, {words} of them in the 32 words ({words / 32:.1f} per word)")
    print(f"edge zeroing (express_zero_edges, static count; its loop over a last unit's pieces runs up to 8 times): {zero}")
    print(f"per-unit scaffolding (unit loop lines, ring wait, refill fast path): {scaffold}")
    print(f"three-class copy (redo after a raised flag): {sum(c3.values())}; general refill (issue): {loop_own['issue (general refill)']}")
    print(f"interior unit: {interior} instructions = {interior / UNIT_BYTES * 1000:.0f} per KB")
    print(f"first / last unit (edge): {edge} instructions = {edge / UNIT_BYTES * 1000:.0f} per KB")
    unit_regions = set(regions) - {"issue (general refill)"} | {"elsewhere"}
    local = [(a, t) for a, r, t in tagged if (s2[0] <= a <= s2[1] or r in unit_regions - {"elsewhere"})
             and re.match(r"(@!?U?P\w+\s+)?(LDL|STL)", t)]
    print(f"LDL / STL in the two-class copy or on the unit loop's lines: {len(local)}")
    for a, t in local:
        print(f"    {a:#06x}  {t}")


if __name__ == "__main__":
    main()
