#!/usr/bin/env python
"""Generate tests/golden/svr.npz by running the UNMODIFIED reference probreg/l2dist_regs.py RigidSVR / TPSSVR and its
features.OneClassSVM on the installed sklearn, loaded as make_golden_l2dist.py loads them.

Every OneClassSVM.compute output (support vectors, weights) is recorded in call order, with the final transformations:
  * the bunny rotated 10 degrees about z with a small translation, at maxiter=1 and maxiter=2 (the second anneals gamma x10);
  * the fish pair, nonrigid (TPSSVR: the constructor's fit, then the registration's two).
Needs a checkout of the reference named by $PROBREG_REFERENCE.   Usage:  python tests/golden/make_golden_svr.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_l2dist as mgl  # noqa: E402


def _recording(features):
    calls = []
    orig = features.OneClassSVM.compute

    def compute(self, data):
        out = orig(self, data)
        calls.append((np.array(out[0]), np.array(out[1]), self._gamma))
        return out

    features.OneClassSVM.compute = compute
    return calls


def _store(out, pre, calls):
    out[pre + "n_calls"] = len(calls)
    for k, (sv, w, g) in enumerate(calls):
        out["%s%d_sv" % (pre, k)], out["%s%d_w" % (pre, k)], out["%s%d_gamma" % (pre, k)] = sv, w, g


def main():
    cf, l2, features = mgl._load()
    calls = _recording(features)
    out = {}
    bunny = np.load(os.path.join(HERE, "bunny.npz"))["source"]
    tgt = bunny.dot(mgl._rot([0.0, 0.0, 1.0], 10.0).T) + [0.01, -0.02, 0.005]
    out["bunny_target"] = tgt
    for maxiter in (1, 2):
        del calls[:]
        reg = l2.RigidSVR(bunny)
        out["bunny_sigma"] = reg._sigma
        res = reg.registration(tgt, maxiter=maxiter)
        pre = "bunny%d_" % maxiter
        _store(out, pre, calls)
        out[pre + "rot"], out[pre + "t"] = res.rot, res.t
    fish_s = np.loadtxt(os.path.join(HERE, "data", "fish_source.txt"))
    fish_t = np.loadtxt(os.path.join(HERE, "data", "fish_target.txt"))
    del calls[:]
    reg = l2.TPSSVR(fish_s)
    out["fish_sigma"] = reg._sigma
    res = reg.registration(fish_t)
    _store(out, "fish_", calls)
    out["fish_a"], out["fish_v"] = res.a, res.v
    np.savez_compressed(os.path.join(HERE, "svr.npz"), **out)
    ang = np.rad2deg(np.arccos((np.trace(out["bunny1_rot"]) - 1.0) / 2.0))
    print("wrote svr.npz: bunny maxiter=1 recovers %.3f of 10 degrees; fish a\n%s" % (ang, out["fish_a"]))


if __name__ == "__main__":
    main()
