#!/usr/bin/env python
"""SASS instructions per pair in the inner loops of the E-step passes.  Usage: sass_pairloop.py lib.so [kernel-substring]

A loop is the range from a backward branch's target to the branch.  Every innermost loop of a pass1_kernel / pass2_kernel
instantiation that issues MUFU.EX2 is a pair loop (one EX2 per pair): its instruction count over its EX2 count is the number of
issue slots a pair costs there, group-sum joins, shared-memory loads and loop control included.  The histogram shows where they go."""
import collections
import re
import subprocess
import sys

lib = sys.argv[1]
want = sys.argv[2] if len(sys.argv) > 2 else "pass"
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout

funcs = collections.OrderedDict()
cur = None
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        funcs[cur] = []
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[T\d]+\s+)?([A-Z0-9_.]+)([^;]*);", line)
    if m and cur:
        funcs[cur].append((int(m.group(1), 16), m.group(2), m.group(3)))

for name, ins in funcs.items():
    if not re.search(r"pass[12]_kernel", name) or want not in name:
        continue
    loops = []
    for addr, op, args in ins:
        t = re.search(r"0x([0-9a-f]+)", args) if op.startswith("BRA") else None
        if t and int(t.group(1), 16) <= addr:
            loops.append((int(t.group(1), 16), addr))
    inner = [(a, b) for a, b in loops if not any((c, d) != (a, b) and a <= c and d <= b for c, d in loops)]
    print(name)
    for a, b in inner:
        body = [op for addr, op, _ in ins if a <= addr <= b]
        ex2 = sum(1 for op in body if op.startswith("MUFU.EX2"))
        if ex2 == 0:
            continue
        hist = collections.Counter(op.split(".")[0] for op in body)
        print("    loop 0x%x-0x%x: %d instructions, %d EX2 -> %.2f per pair   %s"
              % (a, b, len(body), ex2, len(body) / ex2, ", ".join("%s:%d" % kv for kv in hist.most_common(8))))
