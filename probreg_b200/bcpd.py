"""Bayesian Coherent Point Drift -- the API surface of ``probreg.bcpd`` with the registration loop on the H100.

``BayesianCoherentPointDrift.expectation_step`` (reference: bcpd.py:53-72) is the CPD E-step with one weight per source point and
runs in the same two sm_90a passes (``cpd_bcpd_estep``, the ``WGT`` instantiations of the pair kernels), so the M x N matrix the
reference materialises never exists.  ``CombinedBCPD.registration`` keeps the whole loop on the device (``cpd_bcpd_begin/step/get``):
the float32 G^-1, the FP64 M x M precision matrix, its LU (cuSOLVER) and the posterior covariance stay resident, and per iteration
only sigma2 and the moved source (for the reference's nearest-neighbour criterion) come back.  ``CombinedBCPD(low_rank=K)`` replaces
the kernel matrix by a rank-K factorisation built on the device (``cpd_bcpd_lowrank_begin``): no G^-1 and nothing of size M x M, a
K x K M-step, for clouds whose kernel matrix is numerically of low rank (extent up to a few sqrt(c)).  The host M-step below
(``maximization_step`` / ``_maximization_step``, the reference's dense algebra restated, split into the three things it computes) is
kept as public API, and a subclass that overrides it is driven by the host loop.
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
    low_rank -- None (the dense loop) or the rank K of a factorisation G ~= Q Bc Q^T of the inverse-multiquadric kernel matrix
    (c = 1), built on the device by a randomised range finder with ``low_rank_iters`` subspace iterations from ``low_rank_seed``; the
    loop then runs with K x K algebra and nothing of size M x M.  Suited to clouds of extent up to about 3 (in the kernel's units,
    sqrt(c) = 1), where G is numerically of low rank; the dense loop remains for the others.  The host M-step stays dense only.
    """

    def __init__(self, source=None, lmd=2.0, k=1.0e20, gamma=1.0, device=0, low_rank=None, low_rank_iters=2, low_rank_seed=0):
        super(CombinedBCPD, self).__init__(source, device)
        self._tf_type = tf.CombinedTransformation
        self.lmd, self.k, self.gamma = lmd, k, gamma
        if low_rank is not None and (isinstance(low_rank, bool) or not isinstance(low_rank, (int, np.integer)) or low_rank < 1):
            raise ValueError("low_rank must be None or a positive integer, got %r" % (low_rank,))
        self.low_rank, self.low_rank_iters, self.low_rank_seed = low_rank, low_rank_iters, low_rank_seed
        self._check_low_rank()

    def _check_low_rank(self):
        if self.low_rank is not None and not self._has_device_loop():
            raise ValueError("low_rank runs on the device loop only: %s overrides the E- or M-step, which stay dense"
                             % type(self).__name__)

    def _initialize(self, target):
        count, dim = self._source.shape
        start_var = self.gamma * math_utils.squared_kernel_sum(self._source, target, device=self._device)
        identity_map = self._tf_type(np.identity(dim), np.zeros(dim))
        if self.low_rank is not None:
            # nothing of size M x M: the factors are built on the device, and only the diagonal of sigma_mat is kept
            self.gmat = self.gmat_inv = None
            return MstepResult(identity_map, None, np.ones(count), 1.0 / count, start_var)
        self.gmat = math_utils.inverse_multiquadric_kernel(self._source, self._source, device=self._device)
        self.gmat_inv = np.linalg.inv(self.gmat)
        return MstepResult(identity_map, None, np.identity(count), 1.0 / count, start_var)

    def maximization_step(self, target, rigid_trans, estep_res, sigma2_p=None):
        if self.low_rank is not None:
            raise ValueError("the host M-step is dense only: it is not available with low_rank")
        return self._maximization_step(self._source, target, rigid_trans, estep_res, self.gmat_inv, self.lmd, self.k, sigma2_p)

    def _has_device_loop(self):
        # a subclass that brings its own E- or M-step is driven through expectation_step / maximization_step instead
        cls = type(self)
        return (cls.maximization_step is CombinedBCPD.maximization_step and cls._maximization_step is CombinedBCPD._maximization_step
                and cls.expectation_step is BayesianCoherentPointDrift.expectation_step)

    def registration(self, target, w=0.0, maxiter=50, tol=0.001):
        """The loop of the reference (bcpd.py:82-101) with G^-1, the M x M precision matrix, its LU and the posterior covariance
        resident on the GPU (cpd_bcpd_begin / cpd_bcpd_step), or with low_rank the K x K loop (cpd_bcpd_lowrank_begin).  Per iteration the moved source comes back for the reference's
        stopping criterion (mean nearest-neighbour distance, cKDTree on the host), and the transformation only when a callback
        wants it.  Returns the CombinedTransformation in the caller's point order."""
        self._check_low_rank()
        if not self._has_device_loop():
            return super(CombinedBCPD, self).registration(target, w, maxiter, tol)
        assert self._tf_type is not None, "transformation type is None."
        cloud = _points(target)
        state = self._initialize(cloud)
        dim = self._source.shape[1]
        if self._h is None or self._h.dim != dim:
            self._h = _cabi.Handle(dim, device=self._device)
        h = self._h
        h.set_source(self._source)
        h.set_target(cloud)
        if self.low_rank is not None:
            h.bcpd_lowrank_begin(1.0, self.lmd, self.k, state.sigma2, w, self.low_rank, self.low_rank_iters, self.low_rank_seed)
        else:
            h.bcpd_begin(self.gmat_inv, self.lmd, self.k, state.sigma2, w)
        tree = cKDTree(cloud, leafsize=10)
        previous = None
        for it in range(maxiter):
            moved = h.bcpd_get(v=False, moved=True)[5]           # T(y) of the state this iteration starts from (bcpd.py:91)
            h.bcpd_step()
            if self._callbacks:
                current = self._device_transformation(h)
                for notify in self._callbacks:
                    notify(current)
            criterion = math_utils.compute_rmse(moved, tree)
            log.debug("Iteration: {}, Criteria: {}".format(it, criterion))
            if previous is not None and abs(previous - criterion) < tol:
                break
            previous = criterion
        return self._device_transformation(h) if maxiter > 0 else state.transformation

    def _device_transformation(self, h):
        rot, t, scale, _, v = h.bcpd_get()[:5]
        return self._tf_type(rot, t, scale, v)

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
    ``CombinedBCPD`` (lmd, k, gamma, device, low_rank, low_rank_iters, low_rank_seed).  Returns the estimated ``CombinedTransformation``.
    """
    solver = CombinedBCPD(_points(source), **kwargs)
    solver.set_callbacks(list(callbacks))
    return solver.registration(_points(target), w, maxiter, tol)
