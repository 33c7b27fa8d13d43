"""Bayesian Coherent Point Drift -- the API surface of ``probreg.bcpd`` with the E-step on the H100.

What is accelerated is ``BayesianCoherentPointDrift.expectation_step`` (reference: bcpd.py:53-72): it is
the CPD E-step with one weight per source point and runs in the same two sm_90a passes (``cpd_bcpd_estep``, the ``WGT``
instantiations of the pair kernels), so the M x N matrix the reference materialises never exists.  The M-step of ``CombinedBCPD``
(reference: bcpd.py:127-156) is dense M x M linear algebra that the reference itself performs on the host -- two matrix inverses per
iteration -- and is outside the accelerated path; it is restated below, split into the three things it computes, so that
``registration_bcpd`` runs end to end with the reference's signature and returns what the reference returns.
"""
import abc
from collections import namedtuple

import numpy as np
from scipy.spatial import cKDTree
from scipy.special import digamma

from . import _cabi, math_utils
from . import transformation as tf
from .cpd import _points
from .log import log

# field names are API (reference: bcpd.py:17-18)
EstepResult = namedtuple("EstepResult", ["nu_d", "nu", "n_p", "px", "x_hat"])
MstepResult = namedtuple("MstepResult", ["transformation", "u_hat", "sigma_mat", "alpha", "sigma2"])


class BayesianCoherentPointDrift(abc.ABC):
    """Base class: holds the source, the callbacks and the device handle; subclasses supply ``_initialize`` and the M-step.

    source -- (M, D) array or None (``set_source`` later);  device -- CUDA ordinal (an extension over the reference signature)
    """

    def __init__(self, source=None, device=0):
        self._tf_type = None
        self._callbacks = []
        self._device = device
        self._h = None
        self._source = _points(source) if source is not None else None

    def set_callbacks(self, callbacks):
        self._callbacks.extend(callbacks)

    def set_source(self, source):
        self._source = _points(source)

    @abc.abstractmethod
    def _initialize(self, target):
        """-> MstepResult the EM loop starts from."""

    # -- E-step: the GPU part ------------------------------------------------------------------------------------------
    def expectation_step(self, t_source, target, scale, alpha, sigma_mat, sigma2, w=0.0):
        """Posterior responsibilities of BCPD, reduced (reference: bcpd.py:53-72); nothing of size M x N is formed.

        t_source (M, D): the moved source;  scale: similarity scale s;  alpha: (M,) mixing weights or a scalar;
        sigma_mat: posterior covariance of the displacement field, M x M or just its diagonal (only sigma_mm enters);
        sigma2: residual variance;  w: outlier probability.  Returns EstepResult(nu_d (N,), nu (M,), n_p, px (M, D), x_hat (M, D)).
        """
        moved, cloud = np.asarray(t_source), np.asarray(target)
        assert moved.ndim == 2 and cloud.ndim == 2, "source and target must have 2 dimensions."
        count, dim = moved.shape
        if self._h is None or self._h.dim != dim:
            self._h = _cabi.Handle(dim, device=self._device)
        variances = np.asarray(sigma_mat, dtype=np.float64)
        if variances.ndim == 2:
            variances = variances.diagonal().copy()
        weights = np.ascontiguousarray(np.broadcast_to(np.asarray(alpha, dtype=np.float64), (count,)))
        self._h.set_source(moved)
        self._h.set_target(cloud)
        col_mass, row_mass, weighted_targets, total = self._h.bcpd_estep(moved, scale, weights, variances, sigma2, w)
        with np.errstate(divide="ignore", invalid="ignore"):
            barycentres = weighted_targets / row_mass[:, None]      # a source nobody explains gets nan, as in the reference
        return EstepResult(col_mass, row_mass, total, weighted_targets, barycentres)

    def maximization_step(self, target, estep_res, sigma2_p=None):
        return self._maximization_step(self._source, target, estep_res, sigma2_p)

    @staticmethod
    @abc.abstractmethod
    def _maximization_step(source, target, estep_res, sigma2_p=None):
        """-> MstepResult"""

    # -- EM driver ---------------------------------------------------------------------------------------------------------
    def registration(self, target, w=0.0, maxiter=50, tol=0.001):
        """Alternate E- and M-steps at most ``maxiter`` times; stop once the mean nearest-neighbour distance from the moved
        source to the target changes by less than ``tol`` between two iterations (reference: bcpd.py:82-101)."""
        assert self._tf_type is not None, "transformation type is None."
        cloud = _points(target)
        state = self._initialize(cloud)
        tree = cKDTree(cloud, leafsize=10)
        previous = None
        for it in range(maxiter):
            similarity = state.transformation.rigid_trans
            moved = state.transformation.transform(self._source)
            posterior = self.expectation_step(moved, cloud, similarity.scale, state.alpha, state.sigma_mat, state.sigma2, w)
            state = self.maximization_step(cloud, similarity, posterior, state.sigma2)
            for notify in self._callbacks:
                notify(state.transformation)
            criterion = math_utils.compute_rmse(moved, tree)
            log.debug("Iteration: {}, Criteria: {}".format(it, criterion))
            if previous is not None and abs(previous - criterion) < tol:
                break
            previous = criterion
        return state.transformation


def _displacement_posterior(source, pulled_back, nu, gmat_inv, lmd, ratio):
    """Gaussian posterior of the displacement field v given the responsibilities (reference: bcpd.py:131-137):
    covariance (lmd G^-1 + ratio diag(nu))^-1 and mean ratio * cov * diag(nu) * (T^-1(x_hat) - y), coordinate by coordinate."""
    precision = lmd * np.asarray(gmat_inv, dtype=np.float64)       # gmat_inv is float32 (inverse of the float32 kernel matrix)
    precision[np.diag_indices_from(precision)] += ratio * nu
    cov = np.linalg.inv(precision)
    mean = ratio * cov.dot((pulled_back - source) * nu[:, None])
    return cov, mean


def _similarity_from_moments(nu, n_p, x_hat, u_hat, var_term):
    """Weighted Procrustes between the barycentres x_hat and the deformed source u_hat (reference: bcpd.py:140-151)."""
    dim = x_hat.shape[1]
    mean_x, mean_u = nu.dot(x_hat) / n_p, nu.dot(u_hat) / n_p
    dx, du = x_hat - mean_x, u_hat - mean_u
    cross = np.einsum("m,mi,mj->ij", nu, dx, du) / n_p
    spread = np.einsum("m,mi,mj->ij", nu, du, du) / n_p + var_term * np.identity(dim)
    left, _, right_t = np.linalg.svd(cross, full_matrices=True)
    signs = np.ones(dim)
    signs[dim - 1] = np.linalg.det(left.dot(right_t))              # keep a proper rotation
    rot = (left * signs).dot(right_t)
    scale = np.trace(rot.dot(cross)) / np.trace(spread)
    return rot, scale, mean_x - scale * rot.dot(mean_u)


def _residual_variance(target, nu_d, nu, n_p, px, y_hat, scale, var_term):
    """sigma2 of the next iteration (reference: bcpd.py:152-157)."""
    dim = target.shape[1]
    quad_x = nu_d.dot((target * target).sum(axis=1))
    cross = (px * y_hat).sum()
    quad_y = nu.dot((y_hat * y_hat).sum(axis=1))
    return (quad_x - 2.0 * cross + quad_y) / (n_p * dim) + scale * scale * var_term


class CombinedBCPD(BayesianCoherentPointDrift):
    """BCPD with a similarity transform around a non-rigid displacement field (reference: bcpd.py:104-156).

    lmd -- weight of the motion-coherence prior;  k -- Dirichlet concentration of the mixing weights;  gamma -- factor on the
    initial sigma2;  device -- CUDA ordinal (extension).
    """

    def __init__(self, source=None, lmd=2.0, k=1.0e20, gamma=1.0, device=0):
        super(CombinedBCPD, self).__init__(source, device)
        self._tf_type = tf.CombinedTransformation
        self.lmd, self.k, self.gamma = lmd, k, gamma

    def _initialize(self, target):
        count, dim = self._source.shape
        self.gmat = math_utils.inverse_multiquadric_kernel(self._source, self._source, device=self._device)
        self.gmat_inv = np.linalg.inv(self.gmat)
        start_var = self.gamma * math_utils.squared_kernel_sum(self._source, target, device=self._device)
        identity_map = self._tf_type(np.identity(dim), np.zeros(dim))
        return MstepResult(identity_map, None, np.identity(count), 1.0 / count, start_var)

    def maximization_step(self, target, rigid_trans, estep_res, sigma2_p=None):
        return self._maximization_step(self._source, target, rigid_trans, estep_res, self.gmat_inv, self.lmd, self.k, sigma2_p)

    @staticmethod
    def _maximization_step(source, target, rigid_trans, estep_res, gmat_inv, lmd, k, sigma2_p=None):
        """Host-side M-step (dense M x M algebra, like the reference's): displacement posterior, mixing weights, similarity,
        variance -- in that order.  ``ratio`` is scale^2 / sigma2^2 exactly as the reference writes it (bcpd.py:131)."""
        nu_d, nu, n_p, px, x_hat = estep_res
        count = source.shape[0]
        ratio = (rigid_trans.scale / sigma2_p) ** 2
        cov, v_hat = _displacement_posterior(source, rigid_trans.inverse().transform(x_hat), nu, gmat_inv, lmd, ratio)
        u_hat = source + v_hat
        alpha = np.exp(digamma(k + nu) - digamma(k * count + n_p))
        var_term = nu.dot(cov.diagonal()) / n_p
        rot, scale, t = _similarity_from_moments(nu, n_p, x_hat, u_hat, var_term)
        y_hat = rigid_trans.transform(u_hat)                       # still the PREVIOUS similarity, as in the reference
        sigma2 = _residual_variance(target, nu_d, nu, n_p, px, y_hat, scale, var_term)
        return MstepResult(tf.CombinedTransformation(rot, t, scale, v_hat), u_hat, cov, alpha, sigma2)


def registration_bcpd(source, target, w=0.0, maxiter=50, tol=0.001, callbacks=(), **kwargs):
    """One-call BCPD (signature of the reference's ``registration_bcpd``, bcpd.py:159-185).

    source, target: (M, D) / (N, D) arrays (or open3d point clouds);  w: outlier probability;  maxiter / tol: EM budget and the
    tolerance on the nearest-neighbour criterion;  callbacks: callables taking the current transformation;  kwargs go to
    ``CombinedBCPD`` (lmd, k, gamma, device).  Returns the estimated ``CombinedTransformation``.
    """
    solver = CombinedBCPD(_points(source), **kwargs)
    solver.set_callbacks(list(callbacks))
    return solver.registration(_points(target), w, maxiter, tol)
