#!/usr/bin/env python
"""Static SASS digest of the jump kernels in kangaroo_b200/csrc/libkgx.so: for one kernel, find the hot
loop (the innermost backward branch that contains the most IMAD.WIDE) and count opcode classes per loop trip.  The stream
kernel's trip is TWO kangaroo jumps (ping-pong unroll), so counts are also given per jump.

  python scripts/sass_digest.py [kernel-substring ...]       (default: every stream_kernel instantiation)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kangaroo_b200", "csrc", "libkgx.so")


def functions():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    cur, funcs = None, {}
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1); funcs[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", ln)
        if m and cur:
            funcs[cur].append((int(m.group(1), 16), m.group(2).strip()))
    return funcs


def opclass(ins):
    ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
    op = ins.split()[0]
    parts = op.split(".")
    if parts[0] == "IMAD":
        if len(parts) > 1 and parts[1] == "WIDE":
            return "IMAD.WIDE"
        if len(parts) > 1 and parts[1] in ("MOV", "IADD", "SHL", "X", "HI"):
            return "IMAD." + parts[1]
        return "IMAD (32-bit)"
    if parts[0] in ("LDG", "STG", "LDS", "STS", "LDL", "STL", "SHFL", "BRA", "CALL", "IADD3", "LOP3", "SHF", "SEL", "ISETP", "MOV", "DFMA", "DADD"):
        return parts[0] + (".X" if parts[0] == "IADD3" and "X" in parts[1:] else "")
    return parts[0]


def digest(name, ins):
    # loops = backward branches; pick the one whose body holds the most IMAD.WIDE but is innermost (smallest such span > 200 instr)
    addr_index = {a: i for i, (a, _) in enumerate(ins)}
    best = None
    for i, (a, t) in enumerate(ins):
        m = re.search(r"\bBRA(?:\.U)?\s+(?:!?U?P\d+,\s*)?(0x[0-9a-f]+)", t)
        if not m:
            continue
        tgt = int(m.group(1), 16)
        if tgt >= a or tgt not in addr_index:
            continue
        body = ins[addr_index[tgt]:i + 1]
        wide = sum(1 for _, x in body if opclass(x) == "IMAD.WIDE")
        if wide < 100:
            continue
        if best is None or len(body) < len(best):
            best = body
    if best is None:
        return None
    c = collections.Counter(opclass(x) for _, x in best)
    return len(best), c


def main():
    pats = sys.argv[1:] or ["stream_kernel"]
    funcs = functions()
    for name in sorted(funcs):
        if not any(p in name for p in pats):
            continue
        r = digest(name, funcs[name])
        print("== %s  (%d SASS instructions in the function)" % (name, len(funcs[name])))
        if r is None:
            print("   no hot loop found")
            continue
        n, c = r
        jumps = 2 if "stream_kernel" in name else 1
        wide = c.get("IMAD.WIDE", 0)
        other_imad = sum(v for k, v in c.items() if k.startswith("IMAD") and k != "IMAD.WIDE")
        print("   hot loop: %d instructions per trip = %d jump(s): %.1f per jump; IMAD.WIDE %.1f per jump (algorithmic 416), "
              "other IMAD-class %.1f per jump" % (n, jumps, n / jumps, wide / jumps, other_imad / jumps))
        for k, v in c.most_common():
            print("   %-14s %5d   %7.1f / jump" % (k, v, v / jumps))


if __name__ == "__main__":
    main()
