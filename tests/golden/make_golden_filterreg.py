#!/usr/bin/env python
"""Generate tests/golden/filterreg.npz by running the UNMODIFIED reference probreg/filterreg.py, loaded as make_golden.py loads the
reference (a bare parent package, open3d stubbed), with its compiled modules bound to:
  * probreg._permutohedral_lattice -> the reference's own permutohedral.cpp, compiled into oracle/_ref by oracle/permutohedral.mk;
  * probreg._kabsch, probreg._pt2pl -> the float32 restatements of cc/kabsch.cc and cc/point_to_plane.cc in oracle/filterreg_oracle.py
    (pybind11 hands the C++ float32 Eigen matrices);
  * probreg._math.squared_kernel -> make_golden.py's float32 restatement; transforms3d (unused by the rigid path) stubbed.
Records: the bunny (tests/golden/bunny.npz source) rotated 20 degrees and translated, pt2pt (15 iterations) and pt2pl (3: its float32 6 x 6 solve drifts from an FP64 one by up to 1e-3 in 15) (normals: numpy PCA over the 10
nearest neighbours, oriented away from the centroid, saved), update_sigma2 on and off, w 0 and 0.1, tol < 0, and one run to the default tol; the fish in 2-D
(tests/golden/data/fish_*.txt), pt2pt.
Needs a checkout of the reference named by $PROBREG_REFERENCE and oracle/_ref built.   Usage:  python tests/golden/make_golden_filterreg.py
"""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

from oracle import filterreg_oracle as fo  # noqa: E402


class _Lattice(object):
    """probreg._permutohedral_lattice.Permutohedral over the compiled reference: init(p (d x n), with_blur), filter(v (vs x n), start)."""

    def init(self, p, with_blur):
        self._f = np.ascontiguousarray(np.asarray(p, np.float32).T)
        self._blur = bool(with_blur)
        self._size = fo.ref_lattice_size(self._f, self._blur)

    def get_lattice_size(self):
        return self._size

    def filter(self, v, start):
        return fo.ref_filter(self._f, np.asarray(v, np.float32).T, self._blur)[0].T


def _load():
    mg.load_reference()
    lat = types.ModuleType("probreg._permutohedral_lattice")
    lat.Permutohedral = _Lattice
    sys.modules["probreg._permutohedral_lattice"] = lat
    kb = types.ModuleType("probreg._kabsch")
    kb.kabsch, kb.kabsch2d = fo.kabsch_f32, fo.kabsch2d_f32
    sys.modules["probreg._kabsch"] = kb
    pp = types.ModuleType("probreg._pt2pl")
    pp.compute_twist_for_pt2pl = fo.pt2pl_f32
    sys.modules["probreg._pt2pl"] = pp
    sys.modules["probreg._ifgt"] = types.ModuleType("probreg._ifgt")
    t3d = types.ModuleType("transforms3d")
    t3d.quaternions = types.ModuleType("transforms3d.quaternions")
    sys.modules["transforms3d"] = t3d
    sys.modules["transforms3d.quaternions"] = t3d.quaternions
    sys.modules["six"] = sys.modules.get("six") or _six()
    return importlib.import_module("probreg.filterreg")


def _six():
    s = types.ModuleType("six")
    s.add_metaclass = lambda meta: (lambda cls: cls)
    return s


def pca_normals(x, k=10):
    from scipy.spatial import cKDTree
    _, nn = cKDTree(x).query(x, k=k)
    nb = x[nn] - x[nn].mean(1, keepdims=True)
    n = np.linalg.eigh(np.einsum("nki,nkj->nij", nb, nb))[1][:, :, 0]
    return n * np.where(((x - x.mean(0)) * n).sum(1) < 0, -1.0, 1.0)[:, None]     # oriented away from the centroid


def bunny_pair():
    src = np.load(os.path.join(HERE, "bunny.npz"))["source"]
    th = np.deg2rad(20.0)
    rot = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
    return src, src.dot(rot.T) + [0.01, -0.005, 0.003]


def fish_pair():
    return (np.loadtxt(os.path.join(HERE, "data", "fish_source.txt")), np.loadtxt(os.path.join(HERE, "data", "fish_target.txt")))


def cases():
    """(name, source, target, normals or None, kwargs of registration_filterreg)"""
    src, tgt = bunny_pair()
    nrm = pca_normals(tgt)
    out = []
    for obj in ("pt2pt", "pt2pl"):
        for upd in (False, True):
            for w in (0.0, 0.1):
                out.append(("bunny_%s_u%d_w%g" % (obj, upd, w), src, tgt, nrm,
                            dict(objective_type=obj, update_sigma2=upd, w=w, maxiter=15 if obj == "pt2pt" else 3, tol=-1.0)))
    out.append(("bunny_pt2pt_tol", src, tgt, nrm, dict(objective_type="pt2pt", update_sigma2=True, maxiter=50, tol=1e-3)))
    fs, ft = fish_pair()
    for upd in (False, True):
        out.append(("fish_u%d" % upd, fs, ft, None, dict(objective_type="pt2pt", update_sigma2=upd, maxiter=15, tol=-1.0,
                                                          tf_init_params={"rot": np.identity(2), "t": np.zeros(2)})))
    return out


def main():
    frg = _load()
    mu = sys.modules["probreg.math_utils"]
    b, f = bunny_pair(), fish_pair()
    out = {"bunny_normals": cases()[0][3], "bunny_sigma2_init": np.float64(mu.squared_kernel_sum(*b)),
           "fish_sigma2_init": np.float64(mu.squared_kernel_sum(*f))}
    for name, s, t, n, kw in cases():
        calls = []
        res = frg.registration_filterreg(s, t, target_normals=n, callbacks=[lambda tfp: calls.append(1)], **kw)
        out[name + "_rot"] = np.asarray(res.transformation.rot, np.float64)
        out[name + "_t"] = np.asarray(res.transformation.t, np.float64)
        out[name + "_sigma2"] = np.float64(res.sigma2)
        out[name + "_q"] = np.float64(res.q)
        out[name + "_iters"] = np.int64(len(calls))
        print(name, len(calls), res.sigma2, res.q)
    np.savez_compressed(os.path.join(HERE, "filterreg.npz"), **out)


if __name__ == "__main__":
    main()
