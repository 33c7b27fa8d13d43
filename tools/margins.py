#!/usr/bin/env python
"""Measured parity margins on the GPU (what the tolerances of tests/ leave unused): prints max deviations, asserts nothing.
   usage: python tools/margins.py   (needs tests/golden/*.npz; the oracle is the checker)"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import cpd_oracle as orc
from probreg_b200 import cpd, _cabi

F = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
def golden(name):
    return np.load(os.path.join(ROOT, "tests", "golden", name))
def deformed(m, seed=9):
    src, _ = orc.synthetic_pair(m)
    return src, src + 0.03 * np.sin(2 * np.pi * src.dot(F)) + 0.002 * np.random.default_rng(seed).standard_normal(src.shape)

# 1. rigid / affine registrations against the oracle at identical iteration counts
for n, kind, iters, w in [(1500, "rigid", 20, 0.0), (1500, "affine", 20, 0.0), (3000, "rigid", 15, 0.2), (20000, "rigid", 8, 0.1)]:
    src, tgt = orc.synthetic_pair(n, kind)
    res = cpd.registration_cpd(src, tgt, kind, w=w, maxiter=iters, tol=-1.0)
    ref, _ = orc.registration(src, tgt, kind, w=w, maxiter=iters, tol=-1.0)
    lin = res.transformation.rot if kind == "rigid" else res.transformation.b
    print("registration %-6s n=%5d it=%2d w=%.1f: |lin - ref| %.2e  |t - ref| %.2e  sigma2 rel %.2e" % (
        kind, n, iters, w, np.abs(lin - ref.params[0]).max(), np.abs(res.transformation.t - ref.params[1]).max(),
        abs(res.sigma2 - ref.sigma2) / ref.sigma2))
# 2. one E-step element-wise and in aggregate
for n, s2, w in [(3000, 0.02, 0.1), (20000, 1e-3, 0.0), (20000, 1e-4, 0.3)]:
    src, tgt = orc.synthetic_pair(n)
    ts = orc.apply_rigid(src, orc.rot_z(29.0), np.array([0.1, -0.2, 0.3]))
    es = cpd.RigidCPD(src).expectation_step(ts, tgt, s2, w)
    ref = orc.expectation_step(ts, tgt, s2, w) if n <= 3000 else None
    if ref is None:
        from oracle import c_oracle
        ref = c_oracle.expectation_step(ts, tgt, s2, w)
    rel = lambda a, b: np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300 + 1e-12 * np.abs(b).max()))
    print("E-step n=%5d sigma2=%.0e w=%.1f: pt1 rel %.2e  p1 rel %.2e  px max|d|/max|px| %.2e  n_p rel %.2e" % (
        n, s2, w, rel(es.pt1, ref.pt1), rel(es.p1, ref.p1), np.abs(es.px - ref.px).max() / np.abs(ref.px).max(), abs(es.n_p - ref.n_p) / ref.n_p))
# 3. dense non-rigid against the reference fixtures
g = golden("nonrigid.npz")
for tag, sk, tk, it, kw in [("fish15", "fish_source", "fish_target", 15, {"beta": 2.0, "lmd": 2.0}), ("nr12", "nr_source", "nr_target", 12, {"beta": 0.5, "lmd": 1.0})]:
    res = cpd.registration_cpd(g[sk], g[tk], "nonrigid", maxiter=it, tol=-1.0, **kw)
    gm = orc.rbf_kernel_f32(g[sk], g[sk], kw["beta"])
    moved_ref = g[sk] + gm.dot(g[tag + "_w"])
    print("dense non-rigid %-6s: sigma2 rel %.2e  moved max|d|/max|moved| %.2e" % (tag, abs(res.sigma2 - float(g[tag + "_sigma2"])) / float(g[tag + "_sigma2"]),
          np.abs(res.transformation.transform(g[sk]) - moved_ref).max() / np.abs(moved_ref).max()))
# 4. low-rank: factorisation error, low-rank loop vs the oracle on the same G and vs the exact-G oracle, vs the dense device loop
for m, rank, iters, beta, lmd, w in [(2000, 60, 5, 2.0, 2.0, 0.05), (1500, 48, 4, 1.0, 1.5, 0.0)]:
    src, tgt = deformed(m)
    reg = cpd.NonRigidCPD(src, beta=beta, lmd=lmd, low_rank=rank)
    res = reg.registration(tgt, w=w, maxiter=iters, tol=-1.0)
    moved, tfm = reg.moved_source(), res.transformation
    g_lr = tfm.q.dot(tfm.bcore).dot(tfm.q.T)
    gx = orc.rbf_kernel_f32(src, src, beta).astype(np.float64)
    same, _ = orc.registration(src, tgt, "nonrigid", maxiter=iters, tol=-1.0, beta=beta, lmd=lmd, w=w, g=g_lr)
    ref, _ = orc.registration(src, tgt, "nonrigid", maxiter=iters, tol=-1.0, beta=beta, lmd=lmd, w=w)
    print("low-rank m=%d K=%d: |G - QBcQ^T|/|G| %.2e;  vs oracle on the same G: sigma2 rel %.2e moved %.2e;  vs exact-G oracle: sigma2 rel %.2e moved %.2e" % (
        m, rank, np.linalg.norm(gx - g_lr, 2) / np.linalg.norm(gx, 2), abs(res.sigma2 - same.sigma2) / same.sigma2,
        np.abs(moved - (src + g_lr.dot(same.params[0]))).max(), abs(res.sigma2 - ref.sigma2) / ref.sigma2, np.abs(moved - (src + gx.dot(ref.params[0]))).max()))
src, tgt = deformed(6000)
a = cpd.NonRigidCPD(src, beta=2.0, lmd=2.0); ra = a.registration(tgt, maxiter=5, tol=-1.0)
b = cpd.NonRigidCPD(src, beta=2.0, lmd=2.0, low_rank=200); rb = b.registration(tgt, maxiter=5, tol=-1.0)
print("low-rank K=200 vs dense device loop at 6000 points, 5 iterations: sigma2 rel %.2e  moved max|d| %.2e" % (abs(rb.sigma2 - ra.sigma2) / ra.sigma2, np.abs(b.moved_source() - a.moved_source()).max()))
src, tgt = deformed(400)
a = cpd.NonRigidCPD(src, beta=0.5, lmd=1.0); ra = a.registration(tgt, maxiter=4, tol=-1.0)
b = cpd.NonRigidCPD(src, beta=0.5, lmd=1.0, low_rank=450); rb = b.registration(tgt, maxiter=4, tol=-1.0)
print("low-rank K=M=400 vs dense device loop, 4 iterations: sigma2 rel %.2e  moved max|d| %.2e" % (abs(rb.sigma2 - ra.sigma2) / ra.sigma2, np.abs(b.moved_source() - a.moved_source()).max()))
