#!/usr/bin/env python
"""Low-rank BCPD (cpd_bcpd_lowrank_begin, K = 200 by default) at a few sizes M = N, with the card's name and power limit first:
  - the set-up split by device events (cpd_lowrank_setup_times: G X products, orthonormalisations, core), after one warm-up set-up;
  - ms per iteration of cpd_bcpd_step split by cpd_bcpd_step_times (E-step | St and Rt | getrf (K) | getrs (K) | the rest), mean of
    5 steps after 2 warm-up steps;
  - the wall time of one CombinedBCPD(low_rank=K).registration of 20 iterations (set-up, loop and the host's cKDTree criterion);
  - a probe estimate of |G - Q Bc Q^T| / |G| (8 random probes, G x in float64 on the host at M <= 20000);
  - and the dense loop (cpd_bcpd_begin) at the first size for comparison, fed G in place of G^-1 as tools/bcpd_timing.py does.
The source spans 2 units (c = 1: the clouds the low-rank mode is for).   usage: python tools/bcpd_lowrank_timing.py [K] [sizes...]
(default 200 20000 50000 100000 200000); run it twice to see the spread."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from probreg_b200 import _cabi, bcpd, math_utils  # noqa: E402
from probreg_b200.synthetic import synthetic_pair  # noqa: E402
from bcpd_timing import card  # noqa: E402


def pair(n, extent=2.0):
    src, _ = synthetic_pair(n)
    src = src * (extent / np.ptp(src, axis=0).max())
    f = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
    tgt = src + 0.03 * extent * np.sin(2 * np.pi * src.dot(f) / extent)
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)


def probe_error(src, q, bc, probes=8):
    """|G x - Q Bc Q^T x| / |G x| over random x, the largest (G x by float64 rows of G, 500 at a time)"""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((src.shape[0], probes))
    gx = np.empty_like(x)
    for b0 in range(0, src.shape[0], 500):
        d2 = ((src[b0:b0 + 500, None, :] - src[None, :, :]) ** 2).sum(-1)
        gx[b0:b0 + 500] = (1.0 / np.sqrt(d2 + 1.0)).dot(x)
    lx = q.dot(bc.dot(q.T.dot(x)))
    return float((np.linalg.norm(gx - lx, axis=0) / np.linalg.norm(gx, axis=0)).max())


def main():
    args = [int(a) for a in sys.argv[1:]]
    rank = args[0] if args else 200
    sizes = args[1:] or [20000, 50000, 100000, 200000]
    print("card: %s" % card(), flush=True)
    keys = ("estep_ms", "system_ms", "getrf_ms", "getrs_ms", "rest_ms")
    names = ("estep", "St+Rt", "getrf", "getrs", "rest")
    for n in sizes:
        src, tgt = pair(n)
        sigma2 = math_utils.squared_kernel_sum(src, tgt)
        h = _cabi.Handle(3)
        h.set_source(src)
        h.set_target(tgt)
        h.bcpd_lowrank_begin(1.0, 2.0, 1e20, sigma2, 0.05, rank)     # warm-up: module load, first-use self-check
        h.set_profiling(True)
        t0 = time.perf_counter()
        h.bcpd_lowrank_begin(1.0, 2.0, 1e20, sigma2, 0.05, rank)
        t_setup = (time.perf_counter() - t0) * 1e3
        setup = list(h.lowrank_setup_times().values())
        for _ in range(2):
            h.bcpd_step()
        split = dict.fromkeys(keys, 0.0)
        steps, sig = 5, []
        for _ in range(steps):
            sig.append(h.bcpd_step())
            for k, v in h.bcpd_step_times().items():
                split[k] += v / steps
        h.set_profiling(False)
        err = probe_error(src, *h.bcpd_lowrank_factors()) if n <= 20000 else float("nan")
        h.close()
        t0 = time.perf_counter()
        bcpd.CombinedBCPD(src, low_rank=rank).registration(tgt, w=0.05, maxiter=20, tol=-1.0)
        t_reg = time.perf_counter() - t0
        print("M=N=%6d K=%d  set-up %.1f ms wall (%s)  iteration %.2f ms (%s)  registration(20 it) %.2f s  probe |G - QBcQ^T|/|G| %.2g"
              "  sigma2 %.4g" % (n, rank, t_setup, ", ".join("%.1f" % x for x in setup), sum(split.values()),
                                 ", ".join("%s %.2f" % (a, split[k]) for a, k in zip(names, keys)), t_reg, err, sig[-1]), flush=True)
    n = sizes[0]
    src, tgt = pair(n)
    g = math_utils.inverse_multiquadric_kernel(src, src)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_begin(g, 2.0, 1e20, math_utils.squared_kernel_sum(src, tgt), 0.05)
    h.bcpd_step()
    h.set_profiling(True)
    split = dict.fromkeys(keys, 0.0)
    for _ in range(3):
        h.bcpd_step()
        for k, v in h.bcpd_step_times().items():
            split[k] += v / 3
    print("M=N=%6d dense loop: iteration %.2f ms (%s)" % (n, sum(split.values()), ", ".join("%s %.2f" % (k[:-3], split[k]) for k in keys)),
          flush=True)


if __name__ == "__main__":
    main()
