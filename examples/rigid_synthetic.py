#!/usr/bin/env python
"""Rigid CPD of two 100k-point clouds on one H100 (the reference's examples/cpd_rigid_cuda.py, without open3d)."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from probreg_b200 import cpd  # noqa: E402
from probreg_b200.synthetic import synthetic_pair  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
source, target = synthetic_pair(n)
rcpd = cpd.RigidCPD(source)
rcpd.registration(target, maxiter=1)          # first call: CUDA context creation and library load
start = time.time()
tf_param, sigma2, q = rcpd.registration(target, maxiter=50)
print("time: %.3f s" % (time.time() - start))
ang = np.rad2deg(np.arctan2(tf_param.rot[1, 0], tf_param.rot[0, 0]))
print("result: rotation about z %.3f deg, scale %.5f, t %s, sigma2 %.3e" % (ang, tf_param.scale, tf_param.t, sigma2))
