#!/usr/bin/env python
"""BCPD on the device: ms per iteration of cpd_bcpd_step at a few sizes (M = N), split by device events into the E-step, building
the precision matrix, getrf, getrs against the identity and the rest; and, for comparison, one host M-step
(CombinedBCPD._maximization_step, numpy/LAPACK) at the first size.  Prints the card's name and power limit first.

The time of an iteration does not depend on the values of G^-1 (LU with partial pivoting does the same work on any nonsingular
matrix), and the host's float32 inverse of a 20k x 20k matrix alone takes minutes, so the loop is fed the kernel matrix G itself
(symmetric positive definite, so every sigma2 stays positive) in place of its inverse.
usage: python tools/bcpd_timing.py [sizes...]   (default 5000 10000 20000)"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from probreg_b200 import _cabi, bcpd, math_utils  # noqa: E402
from probreg_b200 import transformation as tf  # noqa: E402
from probreg_b200.synthetic import synthetic_pair  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip() or q.stderr.strip()
    except OSError as e:
        return "nvidia-smi unavailable (%s)" % e


def pair(n):
    src, _ = synthetic_pair(n)
    src = src * (n / 1000.0) ** (1.0 / 3.0) * 10.0          # about one unit between neighbours (the IMQ kernel's c = 1)
    f = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
    tgt = np.ascontiguousarray(src + 0.3 * np.sin(2 * np.pi * src.dot(f) / src.max()))
    return np.ascontiguousarray(src), tgt


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [5000, 10000, 20000]
    print("card: %s" % card(), flush=True)
    keys = ("estep_ms", "system_ms", "getrf_ms", "getrs_ms", "rest_ms")
    for n in sizes:
        src, tgt = pair(n)
        g = math_utils.inverse_multiquadric_kernel(src, src)
        sigma2 = math_utils.squared_kernel_sum(src, tgt)
        h = _cabi.Handle(3)
        h.set_source(src)
        h.set_target(tgt)
        t0 = time.perf_counter()
        h.bcpd_begin(g, 2.0, 1e20, sigma2, 0.05)
        t_begin = time.perf_counter() - t0
        h.bcpd_step()                                        # warm-up: module load, solver workspace, first-use paths
        h.set_profiling(True)
        split = dict.fromkeys(keys, 0.0)
        steps, sig = 3, []
        t0 = time.perf_counter()
        for _ in range(steps):
            sig.append(h.bcpd_step())
            for k, v in h.bcpd_step_times().items():
                split[k] += v / steps
        wall = (time.perf_counter() - t0) / steps * 1e3
        h.set_profiling(False)
        print("M=N=%6d  begin %.1f ms, %.1f ms/iteration (wall, profiling on): %s; sigma2 %s" % (
            n, t_begin * 1e3, wall, ", ".join("%s %.2f" % (k[:-3], split[k]) for k in keys), ["%.4g" % s for s in sig]), flush=True)
        if n == sizes[0]:
            # the host loop's M-step on the same pair (one call), after one E-step of the library
            reg = bcpd.CombinedBCPD(src)
            alpha, sdiag = np.full(n, 1.0 / n), np.ones(n)
            es = reg.expectation_step(src, tgt, 1.0, alpha, sdiag, sigma2, 0.05)
            ginv = g.astype(np.float32)
            t0 = time.perf_counter()
            bcpd.CombinedBCPD._maximization_step(src, tgt, tf.RigidTransformation(np.identity(3), np.zeros(3), 1.0), es, ginv, 2.0, 1e20,
                                                 sigma2)
            print("M=N=%6d  host M-step (numpy, %d CPU threads visible): %.1f ms" % (n, os.cpu_count(), (time.perf_counter() - t0) * 1e3),
                  flush=True)
        h.close()


if __name__ == "__main__":
    main()
