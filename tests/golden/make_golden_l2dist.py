#!/usr/bin/env python
"""Generate tests/golden/l2dist.npz by running the UNMODIFIED reference probreg/cost_functions.py, l2dist_regs.py, features.py,
transformation.py and se3_op.py (v0.3.7).

Same loading trick as make_golden.py (a bare parent package, open3d stubbed) plus:
  * ``transforms3d.quaternions.quat2mat`` restated (oracle/l2dist_oracle.py: quat2mat, transforms3d's formula);
  * ``probreg._ifgt.Ifgt`` replaced by the exact float64 direct Gauss transform (the reference switches to IFGT for h >= 0.01);
  * ``probreg._math.tps_kernel_2d`` / ``_3d`` as float32 restatements (oracle/l2dist_oracle.py: tps_kernel).
``features.GMM`` is the reference's own, on the installed sklearn; with ``np.random.seed`` fixed its k-means start is
deterministic.  The fixture holds f and the gradient of both cost functions at several theta, the features the reference computed,
and the results of RigidGMMReg on the bunny and TPSGMMReg on the fish pair; the tests replay those features.
Needs a checkout of the reference named by $PROBREG_REFERENCE.   Usage:  python tests/golden/make_golden_l2dist.py
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

from oracle import l2dist_oracle as lo  # noqa: E402


class _DirectIfgt(object):
    def __init__(self, source, h, eps):
        self._source, self._h = np.asarray(source, dtype=np.float64), h

    def compute(self, target, weights):
        return lo.gauss_transform(np.asarray(target, dtype=np.float64), self._source, self._h, weights)[0]


def _load():
    mg.load_reference()
    t3d = types.ModuleType("transforms3d")
    t3d.quaternions = types.ModuleType("transforms3d.quaternions")
    t3d.quaternions.quat2mat = lo.quat2mat
    sys.modules["transforms3d"] = t3d
    sys.modules["transforms3d.quaternions"] = t3d.quaternions
    ifgt = types.ModuleType("probreg._ifgt")
    ifgt.Ifgt = _DirectIfgt
    sys.modules["probreg._ifgt"] = ifgt
    m = sys.modules["probreg._math"]
    m.tps_kernel_2d = lo.tps_kernel
    m.tps_kernel_3d = lo.tps_kernel
    o3 = sys.modules["open3d"]
    o3.pipelines = types.ModuleType("open3d.pipelines")
    return (importlib.import_module("probreg.cost_functions"), importlib.import_module("probreg.l2dist_regs"),
            importlib.import_module("probreg.features"))


def _recording(features):
    """wrap GMM.compute so that every fit's (means, weights) is kept, in call order"""
    calls = []
    orig = features.GMM.compute

    def compute(self, data):
        out = orig(self, data)
        calls.append((np.array(out[0]), np.array(out[1])))
        return out

    features.GMM.compute = compute
    return calls


def _rot(axis, deg):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.identity(3) + np.sin(th) * k + (1.0 - np.cos(th)) * k.dot(k)


def main():
    cf, l2, features = _load()
    calls = _recording(features)
    out = {}
    rng = np.random.default_rng(5)
    bunny = np.load(os.path.join(HERE, "bunny.npz"))["source"]
    fish_s = np.loadtxt(os.path.join(HERE, "data", "fish_source.txt"))
    fish_t = np.loadtxt(os.path.join(HERE, "data", "fish_target.txt"))
    # 1. the rigid cost at several theta (unit and non-unit quaternions) on synthetic mixtures
    ms = rng.standard_normal((60, 3)) * [0.3, 0.2, 0.1]
    mt = ms.dot(_rot([1, 2, 3], 20.0).T) + [0.05, -0.02, 0.01] + 0.01 * rng.standard_normal(ms.shape)
    ps, pt = rng.dirichlet(np.ones(60)), rng.dirichlet(np.ones(60))
    thetas = np.array([[1.0, 0, 0, 0, 0, 0, 0], [0.9, 0.1, -0.2, 0.3, 0.01, 0.02, -0.03], [0.5, 0.5, 0.5, 0.5, 0.0, 0.1, 0.0],
                       [1.3, -0.2, 0.4, 0.1, -0.05, 0.0, 0.02]])
    rc = cf.RigidCostFunction()
    out["rigid_ms"], out["rigid_ps"], out["rigid_mt"], out["rigid_pt"], out["rigid_sigma"] = ms, ps, mt, pt, 0.15
    out["rigid_thetas"] = thetas
    fg = [rc(th, ms, ps, mt, pt, 0.15) for th in thetas]
    out["rigid_f"], out["rigid_grad"] = np.array([f for f, _ in fg]), np.array([g for _, g in fg])
    # 2. the TPS cost, 2-D and 3-D
    for d in (2, 3):
        ctrl = rng.standard_normal((25, d)) * 0.5
        tms = rng.standard_normal((30, d)) * 0.5
        tmt = tms + 0.05 * rng.standard_normal(tms.shape)
        tps_ = rng.dirichlet(np.ones(30))
        tpt = rng.dirichlet(np.ones(30))
        tc = cf.TPSCostFunction(ctrl, 1.0, 0.1)
        x0 = tc.initial()
        ths = np.array([x0, x0 + 0.01 * rng.standard_normal(x0.shape), x0 + 0.05 * rng.standard_normal(x0.shape)])
        fg = [tc(th, tms, tps_, tmt, tpt, 0.3) for th in ths]
        pre = "tps%d_" % d
        out[pre + "ctrl"], out[pre + "ms"], out[pre + "ps"], out[pre + "mt"], out[pre + "pt"], out[pre + "sigma"] = ctrl, tms, tps_, tmt, tpt, 0.3
        out[pre + "thetas"], out[pre + "f"], out[pre + "grad"] = ths, np.array([f for f, _ in fg]), np.array([g for _, g in fg])
    # 3. RigidGMMReg on the bunny (20 degrees about (1, 1, 0) and a translation), the reference's defaults
    tgt = bunny.dot(_rot([1.0, 1.0, 0.0], 20.0).T) + [0.01, -0.02, 0.005]
    np.random.seed(0)
    del calls[:]
    reg = l2.RigidGMMReg(bunny)
    sigma0 = reg._sigma
    res = reg.registration(tgt)
    out["bunny_target"], out["bunny_sigma"] = tgt, sigma0
    (out["bunny_mu_s"], out["bunny_phi_s"]), (out["bunny_mu_t"], out["bunny_phi_t"]) = calls
    out["bunny_rot"], out["bunny_t"] = res.rot, res.t
    # 4. TPSGMMReg on the fish pair: the constructor's fit (control points), then the registration's two fits
    np.random.seed(1)
    del calls[:]
    reg = l2.TPSGMMReg(fish_s)
    sigma0 = reg._sigma
    res = reg.registration(fish_t)
    out["fish_sigma"] = sigma0
    (out["fish_ctrl"], _), (out["fish_mu_s"], out["fish_phi_s"]), (out["fish_mu_t"], out["fish_phi_t"]) = calls
    out["fish_a"], out["fish_v"] = res.a, res.v
    np.savez_compressed(os.path.join(HERE, "l2dist.npz"), **out)
    print("wrote l2dist.npz: bunny rot\n%s\nfish a\n%s" % (out["bunny_rot"], out["fish_a"]))


if __name__ == "__main__":
    main()
