#!/usr/bin/env python
"""Many small rigid registrations in one call: copies of the bunny (397 points, tests/golden/bunny.npz) at several rotations about
z, each registered back to the original by registration_cpd_batch (one CTA per pair on the GPU)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from probreg_b200 import cpd  # noqa: E402

bunny = np.load(os.path.join(ROOT, "tests", "golden", "bunny.npz"))["source"]
angles = np.arange(-40.0, 41.0, 10.0)
rng = np.random.default_rng(0)
targets = []
for a in np.deg2rad(angles):
    rot = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
    targets.append(bunny.dot(rot.T) + rng.uniform(-0.01, 0.01, 3))
results, n_iter = cpd.registration_cpd_batch([bunny] * len(targets), targets, "rigid")
for deg, res, it in zip(angles, results, n_iter):
    found = np.rad2deg(np.arctan2(res.transformation.rot[1, 0], res.transformation.rot[0, 0]))
    print("rotated %+5.1f deg: found %+8.3f deg in %2d iterations, sigma2 %.3e" % (deg, found, it, res.sigma2))
