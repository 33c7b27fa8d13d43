#!/usr/bin/env python
"""Rigid support vector registration on the bunny -- counterpart of the reference's examples/svr_rigid.py
(l2dist_regs.registration_svr; no open3d viewer: the callback counts BFGS iterations).  The bunny of tests/golden/data, voxel
size 0.005, the target rotated by 10 degrees about z; the reference's single outer iteration."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from probreg_b200 import io, l2dist_regs  # noqa: E402

source = io.voxel_down_sample(io.read_points(os.path.join(ROOT, "tests", "golden", "data", "bunny.pcd")), 0.005)
th = np.deg2rad(10.0)
rot = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
target = source.dot(rot.T)
seen = []
t0 = time.perf_counter()
tf_param = l2dist_regs.registration_svr(source, target, callbacks=[seen.append])
dt = time.perf_counter() - t0
angle = np.rad2deg(np.arctan2(tf_param.rot[1, 0], tf_param.rot[0, 0]))
print("%d points, %d BFGS iterations in %.3f s: rotation about z %.3f deg (truth 10), t %s" % (len(source), len(seen), dt, angle, tf_param.t))
