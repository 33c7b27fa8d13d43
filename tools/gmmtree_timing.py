#!/usr/bin/env python
"""GMMTree at M = N = 100k and 1M for tree_level 2 and 3, with the card's name and power limit first:
  - the build split per level (device events, cpd_gmmtree_times) and the EM iterations each level ran;
  - ms per registration E-step (device events, mean of 5 after 2 warm-up calls);
  - ms of the host M-step (numpy, mean of 5);
  - the wall time of registration_gmmtree over 20 iterations (build included);
  - and, labelled as such, the float64 numpy oracle (oracle/gmmtree_oracle.py, not the reference) at 100k: one registration
    E-step and the first level of the build capped at 3 EM iterations.
The cloud: a few anisotropic Gaussian lumps in a unit box; the target is the source rotated by 10 degrees.
usage: python tools/gmmtree_timing.py [sizes...] (default 100000 1000000)"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from probreg_b200 import _cabi, gmmtree  # noqa: E402
from bcpd_timing import card  # noqa: E402


def cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    centres, scales = rng.uniform(-1.0, 1.0, (5, 3)), rng.uniform(0.05, 0.3, (5, 3))
    lab = rng.integers(0, 5, n)
    src = centres[lab] + rng.standard_normal((n, 3)) * scales[lab]
    th = np.deg2rad(10.0)
    rot = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
    return src, src.dot(rot.T)


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [100000, 1000000]
    print("card: %s" % card(), flush=True)
    for n in sizes:
        src, tgt = cloud(n)
        for levels in (2, 3):
            gt = gmmtree.GMMTree(None, tree_level=levels)
            h = gt._handle()
            h.set_profiling(True)
            t0 = time.perf_counter()
            gt.set_source(src)
            t_build = time.perf_counter() - t0
            lv = h.gmmtree_times()["level_ms"][:levels]
            h.set_target(tgt)
            for _ in range(2):
                h.gmmtree_estep(np.identity(3), np.zeros(3), 0.01)
            es = []
            for _ in range(5):
                mom = h.gmmtree_estep(np.identity(3), np.zeros(3), 0.01)
                es.append(h.gmmtree_times()["estep_ms"])
            res = gmmtree.EstepResult(gmmtree._moment_list(mom))
            t0 = time.perf_counter()
            for _ in range(5):
                gt.maximization_step(res, gt._tf_result)
            t_m = (time.perf_counter() - t0) / 5 * 1e3
            h.set_profiling(False)
            h.close()
            t0 = time.perf_counter()
            gmmtree.registration_gmmtree(src, tgt, maxiter=20, tol=-1.0, tree_level=levels)
            t_reg = time.perf_counter() - t0
            print("M=N=%7d L=%d  build %.3f s wall, per level ms %s, iterations %s  E-step %.3f ms  host M-step %.2f ms  "
                  "registration_gmmtree(20 it) %.3f s" % (n, levels, t_build, ", ".join("%.1f" % x for x in lv),
                                                          list(gt.build_iterations), float(np.mean(es)), t_m, t_reg), flush=True)
        if n <= 100000:
            sys.path.insert(0, ROOT)
            from oracle import gmmtree_oracle as go

            seeds = np.random.default_rng(0).integers(0, n, 64)
            t0 = time.perf_counter()
            go.build(src, 1, 1e-3, 1e-4, seeds[:8], maxiter=3)
            t_ob = time.perf_counter() - t0
            nodes, _, _, _ = go.build(src[:2000], 2, 1e-3, 1e-4, np.random.default_rng(0).integers(0, 2000, 64), maxiter=2)
            t0 = time.perf_counter()
            go.reg_estep(tgt, nodes, 2, 0.01)
            t_oe = time.perf_counter() - t0
            print("M=N=%7d numpy float64 ORACLE (not the reference): level 0 of the build, 3 EM iterations %.3f s; one "
                  "registration E-step (L=2) %.1f ms" % (n, t_ob, t_oe * 1e3), flush=True)


if __name__ == "__main__":
    main()
