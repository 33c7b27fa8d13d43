"""Synthetic workloads of BASELINE.md section 3 (used by bench.py and the examples).

source = anisotropic uniform box; target = permuted, noised (sigma 0.01), transformed copy.
An isotropic blob makes rigid CPD with update_scale collapse towards scale ~0.45 and crawl,
hence the 1.0 x 0.6 x 0.3 box.
"""
import numpy as np


def rot_z(deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def synthetic_pair(n, kind="rigid", noise=0.01, seed=0):
    src = np.random.default_rng(seed).random((n, 3)) * np.array([1.0, 0.6, 0.3])
    rng1 = np.random.default_rng(seed + 1)
    perm = rng1.permutation(n)
    pts = src[perm] + noise * rng1.standard_normal((n, 3))
    lin = rot_z(30.0)
    if kind == "affine":
        lin = lin.dot(np.diag([1.1, 0.9, 1.05]))
        lin[0, 1] += 0.05
    tgt = pts.dot(lin.T) + np.array([0.1, -0.2, 0.3])
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)
