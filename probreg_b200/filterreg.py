"""FilterReg (Gao & Tedrake, CVPR 2019) -- the API surface of ``probreg.filterreg`` with the E-step on the H100.

The E-step filters the target's moments through the reference's permutohedral lattice on the device (``cpd_filterreg_estep``,
csrc/lattice.cuh): the lattice, its blur / no-blur decision and m0, m1, m2 and nx are bit-identical to the reference's x86-64 build
on the same float32 features.  The source is moved in FP64 in a fixed order (x' = ((R00 x + R01 y) + R02 z) + t0, no FMA), so the
features of every iteration are a function of (R, t, sigma2) alone.  The M-step is the reference's (filterreg.py:159-196), in FP64
numpy on the E-step's output.  With the default (identity) ``feature_fn`` the loop runs on the device (``cpd_filterreg_begin /
step``): the clouds are uploaded once, and each iteration moves the source, runs the E-step and reduces the M-step's sums in FP64 on
the GPU; only 49 doubles come back, and the 3 x 3 SVD / 2-D angle / 6 x 6 solve on them stay in numpy.  Any other ``feature_fn`` is
evaluated on the host each iteration and its features are filtered through ``gaussian_filtering.Permutohedral``.

Departures from the reference, on purpose:
  * the M-step (the Kabsch centres and H, the point-to-plane normal equations, q and sigma2) is FP64, where the reference's C++
    runs float32 with OpenMP-order reductions;
  * ``feature_fn`` must return 2 or 3 columns: the lattice is built for d = 2 and 3 (the reference's FPFH features need open3d);
  * ``DeformableKinematicFilterReg`` needs the dq3d package, as in the reference, and raises its RuntimeError.
"""
from collections import namedtuple

import numpy as np

from . import _cabi
from . import math_utils as mu
from . import se3_op as so
from . import transformation as tf
from .log import log

EstepResult = namedtuple("EstepResult", ["m0", "m1", "m2", "nx"])
MstepResult = namedtuple("MstepResult", ["transformation", "sigma2", "q"])
MstepResult.__doc__ = """Result of Maximization step.

    Attributes:
        transformation (tf.Transformation): Transformation from source to target.
        sigma2 (float): Variance of Gaussian distribution.
        q (float): Result of likelihood.
"""


def _points(x):
    return None if x is None else np.asarray(x.points if hasattr(x, "points") else x)


def move(source, rot, t):
    """The source moved in FP64 in a fixed order without FMA: x'_a = ((R_a0 x + R_a1 y) + R_a2 z) + t_a."""
    s = np.asarray(source, np.float64)
    out = np.empty_like(s)
    for a in range(s.shape[1]):
        acc = rot[a, 0] * s[:, 0]
        for b in range(1, s.shape[1]):
            acc = acc + rot[a, b] * s[:, b]
        out[:, a] = acc + t[a]
    return out


def _centres_and_h(model, target, weight):
    tw = weight.sum()
    mc = (weight[:, None] * model).sum(0) / tw
    tc = (weight[:, None] * target).sum(0) / tw
    w2 = weight * weight
    return mc, tc, ((w2[:, None] * (model - mc)).T @ (target - tc)) / w2.sum()


def kabsch(model, target, weight):
    """cc/kabsch.cc:6-56: weighted centres, H weighted by weight^2 over its sum, R = V diag(1, 1, det(UV)) U^T."""
    if weight.sum() == 0:
        return np.identity(3), np.zeros(3)
    mc, tc, hh = _centres_and_h(model, target, weight)
    u, _, vt = np.linalg.svd(hh)
    ss = np.ones(3)
    ss[2] = np.linalg.det(u @ vt.T)
    r = vt.T @ np.diag(ss) @ u.T
    return r, tc - r @ mc


def kabsch2d(model, target, weight):
    """cc/kabsch.cc:58-109: the angle atan2(H01 - H10, H00 + H11)."""
    if weight.sum() == 0:
        return np.identity(2), np.zeros(2)
    mc, tc, hh = _centres_and_h(model, target, weight)
    ang = np.arctan2(hh[0, 1] - hh[1, 0], hh[0, 0] + hh[1, 1])
    r = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    return r, tc - r @ mc


def compute_twist_for_pt2pl(model, target, normal, weight):
    """cc/point_to_plane.cc:6-32: J^T J and J^T r weighted by w, the residual sum by w^2, then the 6 x 6 solve."""
    res = (normal * (target - model)).sum(1)
    jac = np.c_[np.cross(model, normal), normal]
    ata = (weight[:, None] * jac).T @ jac
    atb = (weight * res) @ jac
    return np.linalg.solve(ata, atb), float((weight * weight * res * res).sum())


class FilterReg(object):
    """FilterReg
    FilterReg is similar to CPD, and the speed performance is improved.
    In this algorithm, not only point-to-point alignment but also
    point-to-plane alignment are implemented.

    Args:
        source (numpy.ndarray, optional): Source point cloud data.
        target_normals (numpy.ndarray, optional): Normals of target points.
        sigma2 (Float, optional): Variance parameter. If this variable is None,
            the variance is updated in Mstep.
        update_sigma2 (bool, optional): If this variable is True, Update sigma2 in the registration iteration.
        device (int, optional): CUDA device of the E-step.
    """

    def __init__(self, source=None, target_normals=None, sigma2=None, update_sigma2=False, device=0):
        self._source = source
        self._target_normals = target_normals
        self._sigma2 = sigma2
        self._update_sigma2 = update_sigma2
        self._tf_type = None
        self._tf_result = None
        self._callbacks = []
        self._device = device

    def set_source(self, source):
        self._source = source

    def set_target_normals(self, target_normals):
        self._target_normals = target_normals

    def set_callbacks(self, callbacks):
        self._callbacks = callbacks

    def expectation_step(self, t_source, target, y, sigma2, update_sigma2, objective_type="pt2pt", alpha=0.015):
        """Expectation step (filterreg.py:78-108): the lattice over [t_source; target] / sigma filters the targets' 1, y,
        |y|^2 (update_sigma2) and normals (pt2pl), read at the sources.  float32, as the reference returns them."""
        assert t_source.ndim == 2 and target.ndim == 2, "source and target must have 2 dimensions."
        if objective_type not in ("pt2pt", "pt2pl"):
            raise ValueError("Unknown objective_type: %s." % objective_type)
        if t_source.shape[1] not in (2, 3):
            raise ValueError("the lattice E-step takes features of 2 or 3 columns, got %d (features of higher dimension, such as "
                             "FPFH, are not supported)" % t_source.shape[1])
        if y.shape[1] != t_source.shape[1]:
            raise ValueError("the E-step filters y through a lattice over the features: y must have the features' %d columns, got %d"
                             % (t_source.shape[1], y.shape[1]))
        normals = _points(self._target_normals) if objective_type == "pt2pl" else None
        if objective_type == "pt2pl" and normals is None:
            raise ValueError("pt2pl needs target_normals.")
        m0, m1, m2, nx, _ = _cabi.filterreg_estep(t_source, target, sigma2, update_sigma2, normals, alpha, self._device) \
            if y is target or np.array_equal(y, target) else self._estep_features(t_source, target, y, sigma2, update_sigma2,
                                                                                   normals, alpha)
        return EstepResult(m0, m1, m2, nx)

    def _estep_features(self, fx, fy, y, sigma2, update_sigma2, normals, alpha):
        """The E-step when the features are not the coordinates: the lattice over the features filters the coordinates y."""
        m, n = fx.shape[0], fy.shape[0]
        sigma = np.sqrt(sigma2)
        from .gaussian_filtering import Permutohedral
        fin = np.r_[np.asarray(fx, np.float64) / sigma, np.asarray(fy, np.float64) / sigma]
        ph = Permutohedral(fin, device=self._device)
        if ph.get_lattice_size() > n * alpha:
            ph = Permutohedral(fin, False, device=self._device)
        y = np.asarray(y, np.float64)
        run = lambda v: ph.filter(np.r_[np.zeros((m, v.shape[1])), v])[:m]  # noqa: E731
        m0 = run(np.ones((n, 1))).ravel()
        m1 = run(y)
        m2 = run(np.square(y).sum(axis=1)[:, None]).ravel() if update_sigma2 else None
        nx = run(np.asarray(normals, np.float64)) if normals is not None else None
        return m0, m1, m2, nx, None

    def maximization_step(self, t_source, target, estep_res, w=0.0, objective_type="pt2pt"):
        return self._maximization_step(t_source, target, estep_res, self._tf_result, self._sigma2, w, objective_type=objective_type)

    @staticmethod
    def _maximization_step(t_source, target, estep_res, trans_p, sigma2, w=0.0, objective_type="pt2pt"):
        return None

    def registration(self, target, w=0.0, objective_type="pt2pt", maxiter=50, tol=0.001, min_sigma2=1.0e-4, feature_fn=None):
        assert self._tf_type is not None, "transformation type is None."
        if objective_type not in ("pt2pt", "pt2pl"):
            raise ValueError("Unknown objective_type: %s." % objective_type)
        target = np.asarray(_points(target), np.float64)
        source = np.asarray(_points(self._source), np.float64)
        q = None
        feature_fn = _identity if feature_fn is None else feature_fn
        ftarget = feature_fn(target)
        if np.ndim(ftarget) != 2 or np.shape(ftarget)[1] not in (2, 3):
            raise ValueError("the lattice E-step takes features of 2 or 3 columns, got shape %s (features of higher dimension, such "
                             "as FPFH, are not supported)" % (np.shape(ftarget),))
        if self._sigma2 is None:
            fsource = feature_fn(source)
            self._sigma2 = max(mu.squared_kernel_sum(fsource, ftarget, self._device), min_sigma2)
        loop = None
        if feature_fn is _identity:
            normals = _points(self._target_normals) if objective_type == "pt2pl" else None
            if objective_type == "pt2pl" and normals is None:
                raise ValueError("pt2pl needs target_normals.")
            # the device loop: the clouds stay on the GPU, each step returns the M-step's FP64 sums
            loop = _cabi.FilterRegLoop(source, target, normals, self._update_sigma2, device=self._device)
        self._loop = loop                      # the last registration's device state (its E-step: self._loop.last_estep())
        res = None
        for i in range(maxiter):
            if loop is not None:
                mom = loop.step(np.asarray(self._tf_result.rot, np.float64), np.asarray(self._tf_result.t, np.float64), self._sigma2, w)
                res = self._mstep_from_moments(mom, source.shape[1], self._tf_result, self._sigma2, self._update_sigma2, objective_type)
            else:
                t_source = move(source, np.asarray(self._tf_result.rot, np.float64), np.asarray(self._tf_result.t, np.float64))
                fsource = feature_fn(t_source)
                estep_res = self.expectation_step(fsource, ftarget, target, self._sigma2, self._update_sigma2, objective_type)
                res = self.maximization_step(t_source, target, estep_res, w=w, objective_type=objective_type)
            if res.q is None:
                res = res._replace(q=q)
                break
            self._tf_result = res.transformation
            self._sigma2 = max(res.sigma2, min_sigma2)
            for c in self._callbacks:
                c(self._tf_result)
            log.debug("Iteration: {}, Criteria: {}".format(i, res.q))
            if q is not None and abs(res.q - q) < tol:
                break
            q = res.q
        return res

    @staticmethod
    def _mstep_from_moments(mom, dim, trans_p, sigma2, update_sigma2, objective_type):
        return None


def _identity(x):
    return x


class RigidFilterReg(FilterReg):
    def __init__(self, source=None, target_normals=None, sigma2=None, update_sigma2=False, tf_init_params={}, device=0):
        super(RigidFilterReg, self).__init__(source=source, target_normals=target_normals, sigma2=sigma2, update_sigma2=update_sigma2,
                                             device=device)
        self._tf_type = tf.RigidTransformation
        params = dict(tf_init_params)
        if source is not None and "rot" not in params and np.asarray(_points(source)).shape[1] == 2:
            params.setdefault("rot", np.identity(2))
            params.setdefault("t", np.zeros(2))
        self._tf_result = self._tf_type(**params)

    @staticmethod
    def _maximization_step(t_source, target, estep_res, trans_p, sigma2, w=0.0, objective_type="pt2pt"):
        """filterreg.py:159-196 in FP64."""
        m, dim = t_source.shape
        n = target.shape[0]
        assert dim == 2 or dim == 3, "dim must be 2 or 3."
        m0, m1, m2, nx = [None if a is None else np.asarray(a, np.float64) for a in estep_res]
        c = w / (1.0 - w) * n / m * (2.0 * sigma2 * np.pi) ** (dim / 2.0)
        nonzero_idx = m0 != 0
        if not nonzero_idx.any():
            return MstepResult(trans_p, sigma2, None)
        m0 = m0[nonzero_idx]
        m1 = m1[nonzero_idx]
        t_source_e = t_source[nonzero_idx]
        m1m0 = np.divide(m1.T, m0).T
        m0m0 = m0 / (m0 + c)
        drxdx = np.sqrt(m0m0 * 1.0 / sigma2)
        rot0, t0 = np.asarray(trans_p.rot, np.float64), np.asarray(trans_p.t, np.float64)
        if objective_type == "pt2pt":
            dr, dt = (kabsch2d if dim == 2 else kabsch)(t_source_e, m1m0, drxdx)
            rx = np.multiply(drxdx, (t_source_e - m1m0).T).T
            rot, t = np.dot(dr, rot0), np.dot(t0, dr.T) + dt
            q = np.linalg.norm(rx, ord=2, axis=1).sum()
        elif objective_type == "pt2pl":
            if dim != 3:
                raise ValueError("pt2pl is 3-D only.")
            nxm0 = (nx[nonzero_idx].T / m0).T
            tw, q = compute_twist_for_pt2pl(t_source_e, m1m0, nxm0, drxdx)
            rot, t = so.twist_mul(tw, rot0, t0)
        else:
            raise ValueError("Unknown objective_type: %s." % objective_type)
        if m2 is not None:
            m2 = m2[nonzero_idx]
            sigma2 = ((m0 * np.square(t_source_e).sum(axis=1) - 2.0 * (t_source_e * m1).sum(axis=1) + m2) / (m0 + c)).sum()
            sigma2 /= 3.0 * m0m0.sum()
        return MstepResult(tf.RigidTransformation(rot, t), sigma2, q)


def _mstep_from_moments(mom, dim, trans_p, sigma2, update_sigma2, objective_type):
    """filterreg.py:163-196 from the device's FP64 sums (cpd_filterreg_step): Kabsch / atan2 on the centred H, or the point-to-plane
    6 x 6 solve, q and sigma2."""
    if mom[0] == 0:
        return MstepResult(trans_p, sigma2, None)
    rot0, t0 = np.asarray(trans_p.rot, np.float64), np.asarray(trans_p.t, np.float64)
    if objective_type == "pt2pt":
        mc, tc = mom[2:2 + dim] / mom[1], mom[5:5 + dim] / mom[1]
        hh = mom[12:21].reshape(3, 3)[:dim, :dim] / mom[8]
        if dim == 2:
            ang = np.arctan2(hh[0, 1] - hh[1, 0], hh[0, 0] + hh[1, 1])
            dr = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
        else:
            u, _, vt = np.linalg.svd(hh)
            ss = np.ones(3)
            ss[2] = np.linalg.det(u @ vt.T)
            dr = vt.T @ np.diag(ss) @ u.T
        dt = tc - dr @ mc
        rot, t = np.dot(dr, rot0), np.dot(t0, dr.T) + dt
        q = mom[9]
    else:
        if dim != 3:
            raise ValueError("pt2pl is 3-D only.")
        ata = np.zeros((6, 6))
        ata[np.triu_indices(6)] = mom[21:42]
        ata = ata + np.triu(ata, 1).T
        tw = np.linalg.solve(ata, mom[42:48])
        q = mom[48]
        rot, t = so.twist_mul(tw, rot0, t0)
    if update_sigma2:
        sigma2 = mom[10] / (3.0 * mom[11])
    return MstepResult(tf.RigidTransformation(rot, t), sigma2, q)


RigidFilterReg._mstep_from_moments = staticmethod(_mstep_from_moments)


class DeformableKinematicFilterReg(FilterReg):
    def __init__(self, source=None, skinning_weight=None, sigma2=None):
        raise RuntimeError("No dq3d python package, filterreg deformation model not available.")


def registration_filterreg(source, target, target_normals=None, sigma2=None, update_sigma2=False, w=0, objective_type="pt2pt",
                           maxiter=50, tol=0.001, min_sigma2=1.0e-4, feature_fn=_identity, callbacks=[], **kwargs):
    """FilterReg registration

    Args:
        source (numpy.ndarray): Source point cloud data.
        target (numpy.ndarray): Target point cloud data.
        target_normals (numpy.ndarray, optional): Normal vectors of target point cloud.
        sigma2 (float, optional): Variance of GMM. If `sigma2` is `None`, `sigma2` is automatically updated.
        w (float, optional): Weight of the uniform distribution, 0 < `w` < 1.
        objective_type (str, optional): The type of objective function selected by 'pt2pt' or 'pt2pl'.
        maxitr (int, optional): Maximum number of iterations to EM algorithm.
        tol (float, optional): Tolerance for termination.
        min_sigma2 (float, optional): Minimum variance of GMM.
        feature_fn (function, optional): Feature function returning 2 or 3 columns.
        callback (:obj:`list` of :obj:`function`, optional): Called after each iteration.
            `callback(probreg.Transformation)`

    Keyword Args:
        tf_init_params (dict, optional): Parameters to initialize transformation (for rigid).
        device (int, optional): CUDA device.

    Returns:
        MstepResult: Result of the registration (transformation, sigma2, q)
    """
    frg = RigidFilterReg(_points(source), _points(target_normals), sigma2, update_sigma2, **kwargs)
    frg.set_callbacks(callbacks)
    return frg.registration(_points(target), w=w, objective_type=objective_type, maxiter=maxiter, tol=tol, min_sigma2=min_sigma2,
                            feature_fn=feature_fn)
