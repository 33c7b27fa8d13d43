#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference (probreg v0.3.7).

Needs a checkout of the reference named by $PROBREG_REFERENCE; the fixtures it
writes are committed so that the tests, which never read the reference, can
check both the oracle and the CUDA path against the reference's own outputs.

How the reference is loaded: ``probreg/__init__.py`` imports
every algorithm (and open3d, transforms3d, ... which are absent here), so a bare
parent package is planted in ``sys.modules`` and only ``probreg.cpd`` /
``probreg.transformation`` / ``probreg.math_utils`` / ``probreg.log`` are imported,
unmodified, from the reference tree.  ``open3d`` is stubbed with two empty classes
(it only appears in annotations / isinstance checks) and the pybind11 module
``probreg._math`` (needs Eigen, missing) is replaced by the float32 numpy
restatement in ``oracle/cpd_oracle.py`` (squared_kernel_f32 / rbf_kernel_f32).

Usage:  python tests/golden/make_golden.py
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("PROBREG_REFERENCE", "")
sys.path.insert(0, ROOT)

from oracle import cpd_oracle as orc  # noqa: E402


def load_reference():
    if not os.path.isdir(os.path.join(REF, "probreg")):
        raise SystemExit("reference checkout not found at %s" % REF)
    o3 = types.ModuleType("open3d")
    o3.geometry = types.ModuleType("open3d.geometry")
    o3.utility = types.ModuleType("open3d.utility")
    o3.geometry.PointCloud = type("PointCloud", (), {})
    o3.utility.Vector3dVector = type("Vector3dVector", (), {})
    sys.modules["open3d"] = o3
    sys.modules["open3d.geometry"] = o3.geometry
    sys.modules["open3d.utility"] = o3.utility
    pkg = types.ModuleType("probreg")
    pkg.__path__ = [os.path.join(REF, "probreg")]
    sys.modules["probreg"] = pkg
    m = types.ModuleType("probreg._math")
    m.squared_kernel = orc.squared_kernel_f32
    m.rbf_kernel = orc.rbf_kernel_f32
    sys.modules["probreg._math"] = m
    pkg._math = m
    return importlib.import_module("probreg.cpd"), importlib.import_module("probreg.transformation")


def read_ascii_pcd(path):
    with open(path) as f:
        lines = f.read().splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith("DATA")) + 1
    return np.array([[float(v) for v in l.split()[:3]] for l in lines[start:] if l.strip()])


def run_fixed(cpd, cls, source, target, iters, w=0.0, **kw):
    """registration with tol<0 (never breaks) -> results after exactly `iters` iterations,
    plus the per-iteration (sigma2, q) trace via the callback protocol."""
    obj = cls(source, **kw)
    trace = []
    res = obj.registration(target, w=w, maxiter=iters, tol=-1.0)
    return res


def pack_tf(res):
    tfm = res.transformation
    out = {"sigma2": np.float64(res.sigma2), "q": np.float64(res.q)}
    for name in ("rot", "t", "scale", "b", "w"):
        if hasattr(tfm, name) and getattr(tfm, name) is not None:
            out[name] = np.asarray(getattr(tfm, name), dtype=np.float64)
    return out


def main():
    cpd, tf = load_reference()
    out_dir = HERE
    bunny = read_ascii_pcd(os.path.join(REF, "examples", "bunny.pcd"))
    rz = orc.rot_z(30.0)
    bunny_t = bunny.dot(rz.T)

    # ---- 1. bunny: init, first E-step, rigid/affine registrations
    g = {"source": bunny, "target": bunny_t}
    r = cpd.RigidCPD(bunny)
    ini = r._initialize(bunny_t)
    g["init_sigma2"] = np.float64(ini.sigma2)
    g["init_q"] = np.float64(ini.q)
    es = r.expectation_step(bunny, bunny_t, float(ini.sigma2), 0.0)
    g["e0_pt1"], g["e0_p1"], g["e0_px"], g["e0_np"] = es.pt1, es.p1, es.px, np.float64(es.n_p)
    es = r.expectation_step(bunny, bunny_t, float(ini.sigma2), 0.3)
    g["e0w_pt1"], g["e0w_p1"], g["e0w_px"], g["e0w_np"] = es.pt1, es.p1, es.px, np.float64(es.n_p)
    for tag, cls, iters, w, kw in [
        ("rigid10", cpd.RigidCPD, 10, 0.0, {}),
        ("rigid10_w01", cpd.RigidCPD, 10, 0.1, {}),
        ("rigid10_noscale", cpd.RigidCPD, 10, 0.0, {"update_scale": False}),
        ("affine10", cpd.AffineCPD, 10, 0.0, {}),
    ]:
        kw = dict(kw)
        if cls is not cpd.NonRigidCPD:
            kw["tf_init_params"] = {}
        res = run_fixed(cpd, cls, bunny, bunny_t, iters, w=w, **kw)
        for k, v in pack_tf(res).items():
            g["%s_%s" % (tag, k)] = v
    # default-tolerance runs (iteration count is part of the result)
    for tag, kw in [("rigid_default", {}), ("affine_default", {"tf_type_name": "affine"})]:
        n_it = [0]
        res = cpd.registration_cpd(bunny, bunny_t, callbacks=[lambda t, c=n_it: c.__setitem__(0, c[0] + 1)],
                                   tf_init_params={}, **kw)
        for k, v in pack_tf(res).items():
            g["%s_%s" % (tag, k)] = v
        g["%s_iters" % tag] = np.int64(n_it[0])
    np.savez_compressed(os.path.join(out_dir, "bunny.npz"), **g)

    # ---- 2. synthetic rigid / affine with noise, outliers and w>0 at 1500 pts
    src, tgt = orc.synthetic_pair(1500, "rigid")
    ts_true = orc.apply_rigid(src, orc.rot_z(30.0), np.array([0.1, -0.2, 0.3]))
    for seed in range(7, 100):
        # far outliers whose nearest-source exponent stays clear of float64's denormal band
        # (-708 .. -745.13): there the reference's own K values carry only a few bits, so no
        # implementation can be compared against it element-wise
        rng = np.random.default_rng(seed)
        outl = (rng.random((200, 3)) - 0.5) * 3.0 + tgt.mean(0)
        d2min = ((ts_true[:, None, :] - outl[None, :, :]) ** 2).sum(-1).min(0)
        if not any((((d2min / (2 * s2)) > 690.0) & ((d2min / (2 * s2)) < 760.0)).any() for s2 in (1.0e-4, 3.0e-3)):
            break
    s_seed = seed
    tgt_o = np.ascontiguousarray(np.r_[tgt, outl])
    s = {"source": src, "target": tgt, "target_outl": tgt_o, "outlier_seed": np.int64(s_seed)}
    for tag, cls, target, iters, w, kw in [
        ("rigid20", cpd.RigidCPD, tgt, 20, 0.0, {}),
        ("rigid20_outl_w", cpd.RigidCPD, tgt_o, 20, 0.2, {}),
        ("rigid30_outl_w0", cpd.RigidCPD, tgt_o, 30, 0.0, {}),
    ]:
        res = run_fixed(cpd, cls, src, target, iters, w=w, tf_init_params={}, **kw)
        for k, v in pack_tf(res).items():
            s["%s_%s" % (tag, k)] = v
    srca, tgta = orc.synthetic_pair(1500, "affine")
    s["source_a"], s["target_a"] = srca, tgta
    res = run_fixed(cpd, cpd.AffineCPD, srca, tgta, 20, tf_init_params={})
    for k, v in pack_tf(res).items():
        s["affine20_%s" % k] = v
    # one E-step deep into the regime where columns die (small sigma2, far outliers, w=0)
    r = cpd.RigidCPD(src)
    ts = tf.RigidTransformation(orc.rot_z(30.0), np.array([0.1, -0.2, 0.3])).transform(src)
    assert np.allclose(ts, ts_true)
    for tag, s2, w in [("dead", 1.0e-4, 0.0), ("deadw", 1.0e-4, 0.1), ("mid", 3.0e-3, 0.0)]:
        es = r.expectation_step(ts, tgt_o, s2, w)
        s["es_%s_sigma2" % tag], s["es_%s_w" % tag] = np.float64(s2), np.float64(w)
        s["es_%s_pt1" % tag], s["es_%s_p1" % tag] = es.pt1, es.p1
        s["es_%s_px" % tag], s["es_%s_np" % tag] = es.px, np.float64(es.n_p)
    s["es_tsource"] = ts
    np.savez_compressed(os.path.join(out_dir, "synthetic1500.npz"), **s)

    # ---- 3. non-rigid (dense G) on the 2-D fish and a small 3-D cloud
    fs = np.loadtxt(os.path.join(REF, "examples", "fish_source.txt"))
    ft = np.loadtxt(os.path.join(REF, "examples", "fish_target.txt"))
    n = {"fish_source": fs, "fish_target": ft}
    res = run_fixed(cpd, cpd.NonRigidCPD, fs, ft, 15, beta=2.0, lmd=2.0)
    for k, v in pack_tf(res).items():
        n["fish15_%s" % k] = v
    n["fish_g"] = np.asarray(res.transformation.g)
    res = run_fixed(cpd, cpd.AffineCPD, fs, ft, 15, tf_init_params={})
    for k, v in pack_tf(res).items():
        n["fishaffine15_%s" % k] = v
    res = run_fixed(cpd, cpd.RigidCPD, fs, ft, 15, tf_init_params={})
    for k, v in pack_tf(res).items():
        n["fishrigid15_%s" % k] = v
    s3, _ = orc.synthetic_pair(400, "rigid")
    f = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
    t3 = s3 + 0.03 * np.sin(2 * np.pi * s3.dot(f))
    n["nr_source"], n["nr_target"] = s3, t3
    res = run_fixed(cpd, cpd.NonRigidCPD, s3, t3, 12, beta=0.5, lmd=1.0)
    for k, v in pack_tf(res).items():
        n["nr12_%s" % k] = v
    # constrained non-rigid (cpd.py:306-404): 25 known correspondences, one of them listed twice
    idx = np.random.default_rng(5).choice(400, 25, replace=False)
    idx_s = np.r_[idx, idx[:1]]
    idx_t = np.r_[idx, idx[:1]]
    n["nrc_idx_source"], n["nrc_idx_target"] = idx_s, idx_t
    res = cpd.ConstrainedNonRigidCPD(s3, beta=0.5, lmd=1.0, alpha=1e-2, idx_source=idx_s, idx_target=idx_t).registration(
        t3, maxiter=8, tol=-1.0)
    for k, v in pack_tf(res).items():
        n["nrc8_%s" % k] = v
    np.savez_compressed(os.path.join(out_dir, "nonrigid.npz"), **n)

    # ---- 4. reference's own known-answer test (tests/test_math_utils.py:6-16)
    x = np.arange(15).reshape(5, 3).astype(np.float64)
    ref_mu = importlib.import_module("probreg.math_utils")
    np.savez_compressed(os.path.join(out_dir, "math_utils.npz"), x=x,
                        sks=np.float64(ref_mu.squared_kernel_sum(x, x)),
                        rbf=np.asarray(ref_mu.rbf_kernel(x * 0.1, x * 0.1, 1.0)))
    for f_ in sorted(os.listdir(out_dir)):
        if f_.endswith(".npz"):
            print(f_, os.path.getsize(os.path.join(out_dir, f_)), "bytes")


if __name__ == "__main__":
    main()
