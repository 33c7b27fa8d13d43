"""Time FilterReg on one GPU: the E-step by stage (device events inside cpd_filterreg_estep) and the registration loop, at 10^5 and
10^6 points per cloud (12 Gaussian lumps), at the first iteration's sigma2 (squared_kernel_sum: a blurred lattice of few vertices)
and at min_sigma2 (no blur, many vertices).  For scale, the reference's own lattice E-step (oracle/_ref, built by build() from the
reference's permutohedral.cpp) on this machine's CPU, one thread.  Prints one table; the card, power limit and clock are read in the
same run.   Usage: python tools/filterreg_timing.py [--sizes 100000 1000000] [--reps 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import filterreg_oracle as fo  # noqa: E402
from probreg_b200 import _cabi, filterreg  # noqa: E402

STAGES = ("elevate", "sort", "number+nbrs", "splat", "blur", "slice")


def lumps(count, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((12, 3)) * 0.05
    return centres[rng.integers(0, 12, count)] + rng.standard_normal((count, 3)) * 0.01


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    print("| points | sigma2 | blur | " + " | ".join(STAGES) + " | E-step call ms | reference lattice E-step (CPU) ms |")
    print("|---|---|---|" + "---|" * len(STAGES) + "---|---|")
    for n in a.sizes:
        src = lumps(n, 1)
        th = 0.2
        r = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1.0]])
        tgt = lumps(n, 2).dot(r.T) + 0.01
        first = max(filterreg.mu.squared_kernel_sum(src, tgt), 1e-4)
        for s2 in (first, 1e-4):
            _cabi.filterreg_estep(src, tgt, s2, True)                      # warm-up
            st, calls = [], []
            for _ in range(a.reps):
                ms = np.zeros(6, np.float32)
                t0 = time.perf_counter()
                blur = _cabi.filterreg_estep(src, tgt, s2, True, stage_ms=ms)[4]
                calls.append((time.perf_counter() - t0) * 1e3)
                st.append(ms.copy())
            med = np.median(np.array(st), axis=0)
            ref = "not measured"
            if fo.ref_available():
                t0 = time.perf_counter()
                fo.expectation_step(src, tgt, s2, True, impl="ref")
                ref = "%.0f" % ((time.perf_counter() - t0) * 1e3)
            print("| %d | %.3g | %s | %s | %.1f | %s |" % (n, s2, blur, " | ".join("%.2f" % x for x in med), np.median(calls), ref))
        reg = filterreg.RigidFilterReg(src, None, None, True)
        reg.registration(tgt, maxiter=2, tol=-1.0)
        reg = filterreg.RigidFilterReg(src, None, None, True)
        t0 = time.perf_counter()
        reg.registration(tgt, maxiter=10, tol=-1.0)
        print("loop at %d points: %.1f ms / iteration (10 iterations, pt2pt, update_sigma2)" % (n, (time.perf_counter() - t0) * 100))


if __name__ == "__main__":
    main()
