#!/usr/bin/env python
"""Thin-plate-spline support vector registration on the fish pair -- counterpart of the reference's examples/svr_nonrigid2d.py
(l2dist_regs.registration_svr(..., "nonrigid")).  Prints the mean distance of the moved source to its nearest target point."""
import os
import sys
import time

import numpy as np
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from probreg_b200 import l2dist_regs  # noqa: E402

source = np.loadtxt(os.path.join(ROOT, "tests", "golden", "data", "fish_source.txt"))
target = np.loadtxt(os.path.join(ROOT, "tests", "golden", "data", "fish_target.txt"))
t0 = time.perf_counter()
tf_param = l2dist_regs.registration_svr(source, target, "nonrigid")
dt = time.perf_counter() - t0
tree = cKDTree(target)
print("%d points in %.3f s: mean nearest-target distance %.4f before, %.4f after"
      % (len(source), dt, tree.query(source)[0].mean(), tree.query(tf_param.transform(source))[0].mean()))
