"""TEST INFRASTRUCTURE: build tests/emu/_build/libcpd_b200_emu.so, the CPU emulation of libcpd_b200.so.

The product library needs an H100; the container the CPU test suite runs in has no GPU.  To still execute
the library's host orchestration (csrc/cpd_b200.cu) and its kernels (csrc/kernels.cuh) there, this script

  1. rewrites every  `kernel<<<grid, block, smem, stream>>>(args)`  of cpd_b200.cu into
     `emu::launch("kernel", dim3(grid), dim3(block), smem, stream, [&]() { kernel(args); })`,
  2. compiles the result with g++ against tests/emu/cuda_runtime.h (fibers for the threads of a block,
     host stand-ins for the runtime API, the inline PTX, CUB's radix sort and cuSOLVER's LU).

Only tests load the result (tests/conftest.py: the `emu` fixture).  It is never on the product path: the
package still refuses to work without the real library and a CUDA device.  It models semantics, not speed.
"""
import hashlib
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "probreg_b200", "csrc")
BUILD = os.path.join(HERE, "_build")
OUT = os.path.join(BUILD, "libcpd_b200_emu.so")


def _match_back(text, i, open_c, close_c):
    """text[i] == close_c: index of the matching open_c."""
    depth = 0
    while i >= 0:
        if text[i] == close_c:
            depth += 1
        elif text[i] == open_c:
            depth -= 1
            if depth == 0:
                return i
        i -= 1
    raise ValueError("unbalanced %s%s" % (open_c, close_c))


def _match_fwd(text, i, open_c, close_c):
    depth = 0
    while i < len(text):
        if text[i] == open_c:
            depth += 1
        elif text[i] == close_c:
            depth -= 1
            if depth == 0:
                return i
        i += 1
    raise ValueError("unbalanced %s%s" % (open_c, close_c))


def _split_top(s):
    """split on commas that are not nested in (), <>, [] or {}"""
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    out.append(cur.strip())
    return out


def translate(text):
    """Rewrite CUDA launch syntax into emu::launch calls."""
    out, pos = "", 0
    while True:
        k = text.find("<<<", pos)
        if k < 0:
            return out + text[pos:]
        # kernel expression: identifier, identifier<template args>, or a parenthesised expression
        j = k - 1
        while text[j].isspace():
            j -= 1
        if text[j] == ")":
            start = _match_back(text, j, "(", ")")
        else:
            if text[j] == ">":
                j = _match_back(text, j, "<", ">") - 1
            while re.match(r"[A-Za-z0-9_:]", text[j]):
                j -= 1
            start = j + 1
        kern = text[start:k].strip()
        e = text.find(">>>", k)
        cfg = _split_top(text[k + 3:e])
        while len(cfg) < 4:
            cfg.append("0" if len(cfg) == 2 else "nullptr")
        a0 = text.find("(", e)
        assert text[e + 3:a0].strip() == "", "unexpected text between >>> and (: %r" % text[e + 3:a0]
        a1 = _match_fwd(text, a0, "(", ")")
        args = text[a0 + 1:a1]
        name = re.sub(r"[^A-Za-z0-9_<>, ]", "", kern)
        out += text[pos:start]
        out += 'emu::launch("%s", dim3(%s), dim3(%s), (size_t)(%s), (cudaStream_t)(%s), [&]() { %s(%s); })' % (
            name, cfg[0], cfg[1], cfg[2], cfg[3], kern, args)
        pos = a1 + 1


def build(force=False, verbose=False):
    srcs = [os.path.join(CSRC, "cpd_b200.cu"), os.path.join(CSRC, "kernels.cuh"), os.path.join(ROOT, "include", "cpd_b200.h")]
    srcs += [os.path.join(HERE, f) for f in ("cuda_runtime.h", "emu_device.h", "emu_runtime.cpp", "emu_solver.h", "emu_nccl.h", "build.py",
                                             os.path.join("cub", "device", "device_radix_sort.cuh"))]
    srcs += sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".cu", ".inl")))
    h = hashlib.sha256(os.environ.get("CPD_EMU_CXXFLAGS", "").encode())
    for s in sorted(set(srcs)):
        with open(s, "rb") as f:
            h.update(f.read())
    stamp = os.path.join(BUILD, "stamp")
    os.makedirs(BUILD, exist_ok=True)
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return OUT
    # host sources (the .cu and the .inl files it includes) get their launches rewritten into _build/, which precedes csrc/ on the
    # include path; device headers (.cuh) are compiled as they are
    gen = os.path.join(BUILD, "cpd_b200_emu.cpp")
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".inl")):
            with open(os.path.join(CSRC, name)) as f:
                text = f.read()
            dst = gen if name == "cpd_b200.cu" else os.path.join(BUILD, name)
            with open(dst, "w") as f:
                f.write("// GENERATED by tests/emu/build.py from probreg_b200/csrc/%s -- do not edit\n" % name + translate(text))
    extra = os.environ.get("CPD_EMU_CXXFLAGS", "").split()        # e.g. -DCPD_P1_STAGE=256: emulate a tuning variant
    cmd = ["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w"] + extra + [
           "-I" + HERE, "-I" + BUILD, "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", OUT, gen, os.path.join(HERE, "emu_runtime.cpp"),
           "-ldl", "-lpthread"]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(h.hexdigest())
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
