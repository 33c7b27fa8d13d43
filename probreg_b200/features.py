"""Feature generators of ``probreg.features`` for the L2-distance registrations (reference: features.py), on the H100.

``GMM`` summarises a cloud by a spherical Gaussian mixture: sklearn's ``GaussianMixture(n_components, covariance_type="spherical")``
fit, run on the device (``cpd_gmm_fit``: FP64 EM, fixed-order reductions, bit-identical runs on one device).

Departure from the reference, on purpose: the fit starts from ``init_params="random_from_data"`` seeded by ``seed`` -- the K
points ``np.random.RandomState(seed).choice(N, K, replace=False)``, exactly sklearn's draw for ``random_state=seed`` -- where the
reference runs sklearn's default, an unseeded k-means initialisation.  The device has no k-means, and a seeded start makes every
fit reproducible.  FPFH and the one-class SVM of the reference are not provided.
"""
import abc

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
