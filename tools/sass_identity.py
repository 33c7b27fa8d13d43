#!/usr/bin/env python
"""Per-kernel comparison of the SASS of two builds of libcpd_b200.so (cuobjdump -sass, addresses stripped): which kernels are
byte-identical, which changed, which are new.  The check that a refactor or a new template parameter left the measured kernels
alone.   usage: sass_identity.py old.so new.so [--fold 'ILb0ELb0EEE=ILb0EEE' ...]"""
import hashlib
import re
import subprocess
import sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    table, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            table[cur] = []
        elif cur:
            table[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line))
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest()[:12] for k, v in table.items()}


def demangle(name):
    return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip().split("(")[0]


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    folds = [a.split("=", 1) for a in sys.argv[1:] if "=" in a and not a.startswith("--")]
    old, new = kernels(args[0]), kernels(args[1])
    for a, b in folds:
        new = {k.replace(a, b): v for k, v in new.items()}
    for k in sorted(old):
        verdict = "identical" if new.get(k) == old[k] else ("CHANGED" if k in new else "gone / signature changed")
        print("%-70s %-14s %-14s %s" % (demangle(k)[:70], old[k], new.get(k, "-"), verdict))
    print("new:", ", ".join(sorted(demangle(k) for k in new if k not in old)) or "-")


if __name__ == "__main__":
    main()
