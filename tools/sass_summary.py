#!/usr/bin/env python
"""Opcode summary of the built engine library (cuobjdump -sass), written to profiles/<tag>_sass_summary.txt.
Runs without a GPU.  usage: sass_summary.py <tag>"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "josefine_b200", "csrc", "libjosefine_b200.so")
MEM = re.compile(r"^(LD|ST|ATOM|RED|LDG|STG|LDS|STS|LDL|STL|LDC|CCTL|MEMBAR|FENCE|ERRBAR)")
SYNC = re.compile(r"^(BAR|VOTE|VOTEU|POPC|FLO|BREV|SHFL|MATCH|WARPSYNC)")
TENSOR = re.compile(r"^(UTC|UTMA|HMMA|IMMA|UBLKCP|TCGEN|LDTM|STTM|UTCHMMA|UTCQMMA)")


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "r01b"
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), collections.Counter())
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and cur is not None:
            cur[m.group(1)] += 1
    out = [f"# cuobjdump opcode summary of libjosefine_b200.so (sm_90a), {tag} (tools/sass_summary.py)",
           "# 128-bit global accesses = LDG.E.128 / STG.E.128 (state planes, mailbox units, Instruction FIFO);",
           "# LDS/STS.128 = shared-memory mailboxes and block-table cache; BAR.SYNC = the per-tick barrier;",
           "# POPC = quorum tally, FLO/BREV = __ffs over delivery masks; ATOMG.ADD = the split-launch task ticket,",
           "# LD.ACQUIRE / ST.RELEASE (.STRONG.GPU) = its hand-over flag.", ""]
    for name, c in funcs.items():
        short = re.sub(r"Ev?N2jr.*$", "...", name)
        fmt = lambda rx: ", ".join(f"{k} {v}" for k, v in c.most_common() if rx.match(k)) or "-"
        out += [f"{short}  {sum(c.values())} SASS instructions", f"  memory : {fmt(MEM)}", f"  sync/vote/bit : {fmt(SYNC)}",
                f"  tensor/TMA : {fmt(TENSOR) if fmt(TENSOR) != '-' else 'none (by design: integer state machine, no dense contraction)'}", ""]
    path = os.path.join(ROOT, "profiles", f"{tag}_sass_summary.txt")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write("\n".join(out))
    print(path, len(funcs), "functions")


if __name__ == "__main__":
    main()
