#!/usr/bin/env python
"""SVR on the device, with the card's name and power limit first:
  - the one-class SVM fit (cpd_ocsvm_fit, nu = 0.1, gamma = 1 / (2 sigma^2) with sigma estimated as RigidSVR does) at 20k, 100k
    and 1M points: the whole fit and its SMO iterations, timed with CUDA events on the default stream that the stateless entry
    point launches on, after a warm-up fit;
  - one SMO iteration as (fit capped at 2000 iterations - fit capped at 1000) / 1000, events as above;
  - registration_svr wall time (rigid, one outer iteration) on the bunny (397 points) and at 20k points.
The clouds: a few Gaussian lumps in a unit box; registration targets are the source rotated by 10 degrees about z.
usage: python tools/svr_timing.py"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from probreg_b200 import _cabi, l2dist_regs  # noqa: E402
from bcpd_timing import card  # noqa: E402
from gmmreg_timing import lumps, rot_z  # noqa: E402


def gamma_of(x):
    h = x - x.mean(0)
    sigma = np.power(np.linalg.det(h.T.dot(h) / (len(x) - 1)), 1.0 / (2.0 * x.shape[1]))
    return 1.0 / (2.0 * sigma ** 2)


def fit_ms(x, g, max_iter=None):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    alpha, rho, it = _cabi.ocsvm_fit(x, 0.1, g, max_iter=max_iter)
    b.record()
    b.synchronize()
    return a.elapsed_time(b), it, int((alpha > 0).sum())


def main():
    print(card())
    x = lumps(2000)
    fit_ms(x, gamma_of(x))
    print("| points | SMO iterations | support vectors | fit (ms) | per iteration (us) |")
    print("|---:|---:|---:|---:|---:|")
    for n in (20_000, 100_000, 1_000_000):
        x = lumps(n, 1)
        g = gamma_of(x)
        ms, it, nsv = fit_ms(x, g)
        t1 = fit_ms(x, g, max_iter=1000)[0]
        t2 = fit_ms(x, g, max_iter=2000)[0]
        print("| %d | %d | %d | %.1f | %.2f |" % (n, it, nsv, ms, (t2 - t1) / 1000 * 1e3), flush=True)
    b = np.load(os.path.join(ROOT, "tests", "golden", "bunny.npz"))["source"]
    for name, src in (("bunny (397)", b), ("20k lumps", lumps(20_000, 2))):
        tgt = src.dot(rot_z(10.0).T)
        t0 = time.perf_counter()
        l2dist_regs.registration_svr(src, tgt)
        print("registration_svr %s: %.3f s" % (name, time.perf_counter() - t0), flush=True)


if __name__ == "__main__":
    main()
