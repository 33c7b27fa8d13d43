#!/usr/bin/env python
"""GMMReg on the device, with the card's name and power limit first:
  - the spherical GMM fit (cpd_gmm_fit) at N = 100k and 1M, K = 800: the whole fit (device events on the handle's stream,
    cpd_timer_start / stop) with its EM iterations, and one E/M iteration as (fit of 6 iterations - fit of 1) / 5 with tol < 0;
  - one cpd_l2_dist call at 800 x 800 and 10 000 x 10 000 (host clock around the call, which ends in a device synchronise;
    median of 5 after a warm-up);
  - registration_gmmreg wall time on the bunny (397 points, K = 317) and at 100k points (K = 800);
  - for scale only, sklearn's GaussianMixture fit at 100k points, K = 800, max_iter = 10, on the host: CPU time.
The clouds: a few Gaussian lumps in a unit box; registration targets are the source rotated by 10 degrees.
usage: python tools/gmmreg_timing.py"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from probreg_b200 import _cabi, l2dist_regs  # noqa: E402
from bcpd_timing import card  # noqa: E402


def lumps(n, seed=0):
    rng = np.random.default_rng(seed)
    centres, scales = rng.uniform(-1.0, 1.0, (6, 3)), rng.uniform(0.03, 0.3, (6, 3))
    lab = rng.integers(0, 6, n)
    return centres[lab] + rng.standard_normal((n, 3)) * scales[lab]


def rot_z(deg):
    th = np.deg2rad(deg)
    return np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])


def fit_ms(h, k, seeds, **kw):
    h.timer_start()
    out = h.gmm_fit(k, seeds, **kw)
    return h.timer_stop(), out[3]


def main():
    print("card: %s" % card(), flush=True)
    for n in (100_000, 1_000_000):
        x = lumps(n)
        seeds = np.random.RandomState(0).choice(n, 800, replace=False)
        h = _cabi.Handle(3)
        h.set_source(x)
        fit_ms(h, 800, seeds, max_iter=2, tol=-1.0)                     # warm-up
        ms, it = fit_ms(h, 800, seeds)
        one = min(fit_ms(h, 800, seeds, max_iter=1, tol=-1.0)[0] for _ in range(3))
        six = min(fit_ms(h, 800, seeds, max_iter=6, tol=-1.0)[0] for _ in range(3))
        print("gmm fit N=%d K=800: %d iterations, %.1f ms; one E/M iteration %.3f ms" % (n, it, ms, (six - one) / 5.0), flush=True)
        h.close()
    rng = np.random.default_rng(1)
    for ns in (800, 10_000):
        ms_, mt = rng.standard_normal((ns, 3)), rng.standard_normal((ns, 3))
        ps, pt = np.full(ns, 1.0 / ns), np.full(ns, 1.0 / ns)
        _cabi.l2_dist(ms_, ps, mt, pt, 0.1)
        ts = []
        for _ in range(5):
            t0 = time.perf_counter()
            _cabi.l2_dist(ms_, ps, mt, pt, 0.1)
            ts.append(time.perf_counter() - t0)
        print("l2_dist %d x %d: %.3f ms (host transfers included)" % (ns, ns, 1e3 * np.median(ts)), flush=True)
    bunny = np.load(os.path.join(ROOT, "tests", "golden", "bunny.npz"))["source"]
    for name, src in (("bunny", bunny), ("100k", lumps(100_000, 2))):
        tgt = src.dot(rot_z(10.0).T)
        t0 = time.perf_counter()
        res = l2dist_regs.registration_gmmreg(src, tgt)
        dt = time.perf_counter() - t0
        ang = np.rad2deg(np.arccos(np.clip((np.trace(res.rot.T.dot(rot_z(10.0))) - 1.0) / 2.0, -1.0, 1.0)))
        print("registration_gmmreg %s (%d points): %.3f s wall, rotation error %.3f deg" % (name, len(src), dt, ang), flush=True)
    try:
        from sklearn.mixture import GaussianMixture
    except ImportError:
        print("sklearn: not installed, not measured")
        return
    x = lumps(100_000)
    t0 = time.perf_counter()
    g = GaussianMixture(800, covariance_type="spherical", init_params="random_from_data", random_state=0, max_iter=10).fit(x)
    print("CPU time, sklearn GaussianMixture fit on the host, N=100k K=800, %d iterations: %.2f s (%d host CPUs)"
          % (g.n_iter_, time.perf_counter() - t0, os.cpu_count()), flush=True)


if __name__ == "__main__":
    main()
