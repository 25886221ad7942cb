#!/usr/bin/env python3
"""Memory-instruction census of the placement kernels in a built libmmplace.so, from its SASS (no GPU needed).

For every kernel whose name matches one of the patterns (default: the lane kernels) it prints registers, stack frame and
static shared memory (cuobjdump -res-usage) and the number of memory instructions by kind in its SASS:
generic LD / ST, local LDL / STL, shared LDS / STS, global LDG / STG.  Generic accesses go through address-space
resolution and cannot use the read-only path; local ones are the stack frame (spills, or an addressable local object).
Spill bytes are not recorded in the binary: pass the compiler's `-Xptxas -v` output with --ptxas-log to add them
(`python -m modelmesh_b200.build --force -v 2> ptxas.log`).

    python tools/sass_census.py [--lib modelmesh_b200/csrc/libmmplace.so] [--ptxas-log ptxas.log] [pattern ...]
"""
from __future__ import annotations

import argparse
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "modelmesh_b200", "csrc", "libmmplace.so")
DEFAULT_PATTERNS = ["k_place_direct", "k_place_lanes", "k_place_small", "k_place_server", "k_place_dealt"]
KINDS = ["LD", "ST", "LDL", "STL", "LDS", "STS", "LDG", "STG"]
OPCODE = re.compile(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P[0-9T]+\s+)?([A-Z0-9_]+)")


def tool(name: str) -> str:
    for cand in (shutil.which(name), os.path.join("/usr/local/cuda/bin", name)):
        if cand and os.path.exists(cand):
            return cand
    raise SystemExit(f"{name} not found")


def demangle(names):
    try:
        out = subprocess.run([tool("cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True).stdout
        return dict(zip(names, out.splitlines()))
    except (SystemExit, subprocess.CalledProcessError):
        return {n: n for n in names}


def sass_counts(lib: str):
    """mangled function name -> {kind: count} over its SASS."""
    text = subprocess.run([tool("cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    counts, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = counts.setdefault(m.group(1), dict.fromkeys(KINDS, 0))
            continue
        m = OPCODE.match(line)
        if cur is not None and m:
            op = m.group(1)
            if op in cur:
                cur[op] += 1
    return counts


def res_usage(lib: str):
    """mangled function name -> (registers, stack bytes, static shared bytes)."""
    text = subprocess.run([tool("cuobjdump"), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
        if cur and m:
            res[cur] = tuple(int(x) for x in m.groups())
    return res


def spills(log: str):
    """mangled function name -> (spill store bytes, spill load bytes), from -Xptxas -v output."""
    out, cur = {}, None
    with open(log) as f:
        for line in f:
            m = re.search(r"Compiling entry function '(\S+)'", line) or re.search(r"Function properties for (\S+)", line)
            if m:
                cur = m.group(1)
                continue
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if cur and m:
                out[cur] = (int(m.group(1)), int(m.group(2)))
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib", default=DEFAULT_LIB)
    ap.add_argument("--ptxas-log", help="-Xptxas -v output of the build that made --lib: adds spill bytes")
    ap.add_argument("patterns", nargs="*", default=DEFAULT_PATTERNS, help="substrings of the demangled kernel names")
    args = ap.parse_args()
    counts, res = sass_counts(args.lib), res_usage(args.lib)
    sp = spills(args.ptxas_log) if args.ptxas_log else {}
    names = demangle(sorted(counts))
    rows = []
    for mangled, c in counts.items():
        short = re.sub(r"\((?:int|bool)\)", "", names.get(mangled, mangled))  # void k<(int)4, (int)6>(...) -> k<4, 6>
        short = short.removeprefix("void ").split("(")[0]
        if not any(p in short for p in args.patterns):
            continue
        reg, stack, shared = res.get(mangled, (None, None, None))
        s = sp.get(mangled)
        rows.append((short, reg, stack, f"{s[0]} / {s[1]}" if s else "-", c, shared))
    if not rows:
        print("no kernel matches", args.patterns, file=sys.stderr)
        return 1
    head = ["kernel", "regs", "stack B", "spill st / ld B", "LD / ST", "LDL / STL", "LDS / STS", "LDG / STG", "smem B"]
    print("| " + " | ".join(head) + " |")
    print("|" + "---|" * len(head))
    for short, reg, stack, s, c, shared in sorted(rows):
        print(f"| `{short}` | {reg} | {stack} | {s} | {c['LD']} / {c['ST']} | {c['LDL']} / {c['STL']} | "
              f"{c['LDS']} / {c['STS']} | {c['LDG']} / {c['STG']} | {shared} |")
    return 0


if __name__ == "__main__":
    sys.exit(main())
