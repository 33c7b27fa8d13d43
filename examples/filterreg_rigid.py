"""FilterReg on the bunny: point-to-point and point-to-plane, E-step on the GPU."""
import os

import numpy as np

from probreg_b200 import filterreg

HERE = os.path.dirname(os.path.abspath(__file__))
bunny = np.load(os.path.join(HERE, "..", "tests", "golden", "bunny.npz"))
source = bunny["source"]
th = np.deg2rad(20.0)
rot = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
target = source.dot(rot.T) + [0.005, 0.0, -0.003]

# normals of the target from a PCA over its 10 nearest neighbours
from scipy.spatial import cKDTree  # noqa: E402

_, nn = cKDTree(target).query(target, k=10)
cov = np.einsum("nki,nkj->nij", target[nn] - target[nn].mean(1, keepdims=True), target[nn] - target[nn].mean(1, keepdims=True))
normals = np.linalg.eigh(cov)[1][:, :, 0]

for objective in ("pt2pt", "pt2pl"):
    res = filterreg.registration_filterreg(source, target, target_normals=normals, objective_type=objective, update_sigma2=True)
    err = np.rad2deg(np.arccos(np.clip((np.trace(res.transformation.rot.T @ rot) - 1) / 2, -1, 1)))
    print("%s: rotation error %.3f deg, sigma2 %.3g, q %.4g" % (objective, err, res.sigma2, res.q))
