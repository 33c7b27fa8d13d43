#!/usr/bin/env python
"""BCPD (similarity + non-rigid) on the GPU -- counterpart of the reference's examples/bcpd_nonrigid.py on a synthetic pair (no
open3d / transforms3d needed).  The whole loop runs on the device (the M x M precision matrix and its LU included); what stays on
the host is the one-off float32 inverse of the kernel matrix (CombinedBCPD._initialize, as in the reference) and the
nearest-neighbour stopping criterion.  The device keeps about 20 M^2 bytes.  With a third argument K the loop runs on a rank-K
factorisation of the kernel matrix instead (CombinedBCPD(low_rank=K)): nothing of size M x M on the device or the host.
usage: python examples/bcpd_nonrigid.py [points] [iters] [low_rank]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from probreg_b200 import bcpd
from probreg_b200.synthetic import synthetic_pair

n = int(sys.argv[1]) if len(sys.argv) > 1 else 5000
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
low_rank = int(sys.argv[3]) if len(sys.argv) > 3 else None
source, target = synthetic_pair(n)
f = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
target = target + 0.01 * np.sin(2 * np.pi * target.dot(f))
# (the reference's BCPD is fragile on unnormalised clouds -- its sigma2 update can overshoot below zero after a few more
#  iterations on this pair, with either implementation; tests/golden/bcpd.npz pins the first five against the reference)
tf_param = bcpd.registration_bcpd(source, target, w=0.05, maxiter=iters, tol=-1.0, low_rank=low_rank)
ang = np.rad2deg(np.arctan2(tf_param.rigid_trans.rot[1, 0], tf_param.rigid_trans.rot[0, 0]))
print("result: rotation about z %.2f deg, scale %.4f, t %s" % (ang, tf_param.rigid_trans.scale, tf_param.rigid_trans.t))
print("mean |v| of the non-rigid part: %.4f" % np.linalg.norm(tf_param.v, axis=1).mean())
