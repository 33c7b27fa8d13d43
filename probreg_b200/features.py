"""Feature generators of ``probreg.features`` for the L2-distance registrations (reference: features.py), on the H100.

``GMM`` summarises a cloud by a spherical Gaussian mixture: sklearn's ``GaussianMixture(n_components, covariance_type="spherical")``
fit, run on the device (``cpd_gmm_fit``: FP64 EM, fixed-order reductions, bit-identical runs on one device).

Departure from the reference, on purpose: the fit starts from ``init_params="random_from_data"`` seeded by ``seed`` -- the K
points ``np.random.RandomState(seed).choice(N, K, replace=False)``, exactly sklearn's draw for ``random_state=seed`` -- where the
reference runs sklearn's default, an unseeded k-means initialisation.  The device has no k-means, and a seeded start makes every
fit reproducible.

``OneClassSVM`` summarises a cloud by the support vectors of sklearn's ``OneClassSVM(kernel="rbf", nu, gamma)`` fit, run on the
device (``cpd_ocsvm_fit``): libsvm's SMO on sklearn's path, so the same support vectors and weights as the reference's fit.  It has
no shrinking (where measured, sklearn's shrinking gives the same weights) and keeps libsvm's float32 rounding of the kernel values
on purpose, since the badly conditioned dual would otherwise end on other weights.  FPFH is not provided.
"""
import abc
import warnings

import numpy as np

from . import _cabi


class Feature(abc.ABC):
    @abc.abstractmethod
    def init(self):
        pass

    @abc.abstractmethod
    def compute(self, data):
        return None

    def annealing(self):
        pass

    def __call__(self, data):
        return self.compute(data)


class GMM(Feature):
    """Feature points extraction using Gaussian mixture model

    n_gmm_components -- the number of mixture components.  Extensions over the reference: seed (of the random_from_data start),
    device (CUDA ordinal), max_iter, tol, reg_covar (sklearn's defaults).  After ``compute``: ``means_``, ``weights_``,
    ``covariances_`` (spherical variances), ``n_iter_`` and ``lower_bounds_`` (one per EM iteration), as sklearn names them.
    """

    def __init__(self, n_gmm_components=800, seed=0, device=0, max_iter=100, tol=1.0e-3, reg_covar=1.0e-6):
        self._n_gmm_components = n_gmm_components
        self._seed = seed
        self._device = device
        self._max_iter = max_iter
        self._tol = tol
        self._reg_covar = reg_covar

    def init(self):
        pass

    def seeds(self, n_points):
        """the K point indices the fit starts from (sklearn's random_from_data draw for random_state=seed)"""
        return np.random.RandomState(self._seed).choice(n_points, self._n_gmm_components, replace=False)

    def compute(self, data):
        x = _cabi.as_cloud(data)
        h = _cabi.Handle(x.shape[1], self._device)
        try:
            h.set_source(x)
            w, mu, var, it, lb = h.gmm_fit(self._n_gmm_components, self.seeds(len(x)), self._reg_covar, self._tol, self._max_iter)
        finally:
            h.close()
        self.weights_, self.means_, self.covariances_, self.n_iter_, self.lower_bounds_ = w, mu, var, it, lb
        return mu, w


class ConvergenceWarning(UserWarning):
    """the one-class SVM fit reached max_iter before its stop test held (sklearn warns with its own ConvergenceWarning)"""


class OneClassSVM(Feature):
    """Feature points extraction using One class SVM

    dim -- dimension of the points; sigma -- width of the Gaussians the support vectors become (weights alpha (2 pi sigma^2)^(D/2));
    gamma -- coefficient of the RBF kernel; nu -- sklearn's nu, in (0, 1]; delta -- annealing factor of gamma.  Extensions over the
    reference: device (CUDA ordinal), tol (of the stop test), max_iter (SMO iterations; None: libsvm's max(10^7, 100 N)).  After
    ``compute``, as sklearn names them: ``support_``, ``support_vectors_``, ``dual_coef_`` (1 x nSV), ``intercept_`` (-rho),
    ``offset_`` (rho) and ``n_iter_``.
    """

    def __init__(self, dim, sigma, gamma=0.5, nu=0.05, delta=10.0, device=0, tol=1.0e-3, max_iter=None):
        self._dim = dim
        self._sigma = sigma
        self._gamma = gamma
        self._nu = nu
        self._delta = delta
        self._device = device
        self._tol = tol
        self._max_iter = max_iter

    def init(self):
        pass

    def compute(self, data):
        x = _cabi.as_cloud(data, self._dim)
        max_iter = max(10_000_000, 100 * len(x)) if self._max_iter is None else self._max_iter
        alpha, rho, it = _cabi.ocsvm_fit(x, self._nu, self._gamma, self._tol, max_iter, self._device)
        if not np.isfinite(rho):
            raise ValueError("The dual coefficients or intercepts are not finite (every alpha is at its bound 1: nu = %g)" % self._nu)
        if it >= max_iter:
            warnings.warn("the one-class SVM fit stopped at max_iter = %d before converging" % max_iter, ConvergenceWarning)
        self.support_ = np.nonzero(alpha > 0.0)[0].astype(np.int32)
        self.support_vectors_ = x[self.support_]
        self.dual_coef_ = alpha[self.support_][None, :]
        self.intercept_ = np.array([-rho])
        self.offset_ = np.array([rho])
        self.n_iter_ = it
        z = np.power(2.0 * np.pi * self._sigma ** 2, self._dim * 0.5)
        return self.support_vectors_, self.dual_coef_[0] * z

    def annealing(self):
        self._gamma *= self._delta
