"""GMMReg (Jian & Vemuri, PAMI 2011) -- the API surface of ``probreg.l2dist_regs`` with the hot paths on the H100.

Each cloud is summarised by a spherical Gaussian mixture (``features.GMM``: the EM fit on the device, ``cpd_gmm_fit``), and the
transformation minimises the L2 distance between the two mixtures with scipy's BFGS (``jac=True``), each evaluation one device
call for the distance and its gradient (``cost_functions``, ``cpd_l2_dist``).  ``registration`` follows l2dist_regs.py:71-97:
per outer iteration new features, a BFGS solve from the last solution, then sigma *= delta.

Departures from the reference, on purpose:
  * the mixtures are seeded ``random_from_data`` fits (``seed``), not sklearn's unseeded k-means start (see ``features``);
  * the Gauss transforms of the L2 distance are exact FP64 sums, not a float32 IFGT;
  * ``TPSGMMReg`` fits the source once, in the constructor, and its means are both the control points and the source mixture of
    every outer iteration: the reference fits it again each time, which with a seeded start gives the same mixture.

Support vector registration (``RigidSVR``, ``TPSSVR``, ``registration_svr``) summarises each cloud by the support vectors of a
one-class SVM (``features.OneClassSVM``: the SMO fit on the device, ``cpd_ocsvm_fit``, on sklearn's path) and minimises the same
L2 distance.  The kernel's gamma is annealed by x10 per outer iteration, so ``TPSSVR`` fits the source again in every outer
iteration after the first; its control points are the support vectors of the constructor's fit, as in the reference.
"""
import logging

import numpy as np
from scipy.optimize import minimize

from . import cost_functions as cf
from . import features as ft
from .log import log


class L2DistRegistration(object):
    """L2 distance registration: both clouds as Gaussian mixtures (feature_gen), the transformation that minimises the L2
    distance between them (cost_fn).  sigma -- scale of the L2 distance; delta -- its annealing factor per outer iteration;
    use_estimated_sigma -- sigma = det(cov(source))^(1 / 2D) instead of the argument."""

    def __init__(self, source, feature_gen, cost_fn, sigma=1.0, delta=0.9, use_estimated_sigma=True):
        self._source = source
        self._feature_gen = feature_gen
        self._cost_fn = cost_fn
        self._sigma = sigma
        self._delta = delta
        self._use_estimated_sigma = use_estimated_sigma
        self._callbacks = []
        if self._source is not None and self._use_estimated_sigma:
            self._estimate_sigma(self._source)

    def set_source(self, source):
        self._source = source
        if self._use_estimated_sigma:
            self._estimate_sigma(self._source)

    def set_callbacks(self, callbacks):
        self._callbacks.extend(callbacks)

    def _estimate_sigma(self, data):
        ndata, dim = data.shape
        data_hat = data - np.mean(data, axis=0)
        self._sigma = np.power(np.linalg.det(np.dot(data_hat.T, data_hat) / (ndata - 1)), 1.0 / (2.0 * dim))

    def _annealing(self):
        self._sigma *= self._delta

    def _source_features(self):
        return self._feature_gen.compute(self._source)

    def optimization_cb(self, x):
        tf_result = self._cost_fn.to_transformation(x)
        for c in self._callbacks:
            c(tf_result)

    def registration(self, target, maxiter=1, tol=1.0e-3, opt_maxiter=50, opt_tol=1.0e-3):
        """Outer loop of l2dist_regs.py:71-97; returns the transformation from source to target."""
        f = None
        x_ini = self._cost_fn.initial()
        for _ in range(maxiter):
            self._feature_gen.init()
            mu_source, phi_source = self._source_features()
            mu_target, phi_target = self._feature_gen.compute(target)
            args = (mu_source, phi_source, mu_target, phi_target, self._sigma)
            res = minimize(self._cost_fn, x_ini, args=args, method="BFGS", jac=True, tol=opt_tol,
                           options={"maxiter": opt_maxiter, "disp": log.level == logging.DEBUG}, callback=self.optimization_cb)
            self._annealing()
            self._feature_gen.annealing()
            if f is not None and abs(res.fun - f) < tol:
                break
            f = res.fun
            x_ini = res.x
        return self._cost_fn.to_transformation(res.x)


class RigidGMMReg(L2DistRegistration):
    """Rigid GMMReg.  Extensions over the reference: seed (of the mixture fits), device (CUDA ordinal)."""

    def __init__(self, source, sigma=1.0, delta=0.9, n_gmm_components=800, use_estimated_sigma=True, seed=0, device=0):
        n_gmm_components = min(n_gmm_components, int(source.shape[0] * 0.8))
        super(RigidGMMReg, self).__init__(source, ft.GMM(n_gmm_components, seed=seed, device=device), cf.RigidCostFunction(device),
                                          sigma, delta, use_estimated_sigma)


class TPSGMMReg(L2DistRegistration):
    """Thin-plate-spline GMMReg: the source mixture's means are the spline's control points.  Extensions over the reference:
    seed, device."""

    def __init__(self, source, sigma=1.0, delta=0.9, n_gmm_components=800, alpha=1.0, beta=0.1, use_estimated_sigma=True, seed=0,
                 device=0):
        n_gmm_components = min(n_gmm_components, int(source.shape[0] * 0.8))
        super(TPSGMMReg, self).__init__(source, ft.GMM(n_gmm_components, seed=seed, device=device),
                                        cf.TPSCostFunction([], alpha, beta, device), sigma, delta, use_estimated_sigma)
        self._feature_gen.init()
        self._src_features = self._feature_gen.compute(source)
        self._cost_fn._control_pts = self._src_features[0]

    def _source_features(self):
        return self._src_features


class RigidSVR(L2DistRegistration):
    """Rigid support vector registration.  Extension over the reference: device (CUDA ordinal)."""

    def __init__(self, source, sigma=1.0, delta=0.9, gamma=0.5, nu=0.1, use_estimated_sigma=True, device=0):
        super(RigidSVR, self).__init__(source, ft.OneClassSVM(source.shape[1], sigma, gamma, nu, device=device),
                                       cf.RigidCostFunction(device), sigma, delta, use_estimated_sigma)

    def _estimate_sigma(self, data):
        super(RigidSVR, self)._estimate_sigma(data)
        self._feature_gen._sigma = self._sigma
        self._feature_gen._gamma = 1.0 / (2.0 * np.square(self._sigma))


class TPSSVR(L2DistRegistration):
    """Thin-plate-spline support vector registration: the support vectors of the source's first fit are the spline's control
    points.  Extension over the reference: device."""

    def __init__(self, source, sigma=1.0, delta=0.9, gamma=0.5, nu=0.1, alpha=1.0, beta=0.1, use_estimated_sigma=True, device=0):
        super(TPSSVR, self).__init__(source, ft.OneClassSVM(source.shape[1], sigma, gamma, nu, device=device),
                                     cf.TPSCostFunction([], alpha, beta, device), sigma, delta, use_estimated_sigma)
        self._feature_gen.init()
        self._first_features = self._feature_gen.compute(source)
        self._cost_fn._control_pts = self._first_features[0]

    def _estimate_sigma(self, data):
        super(TPSSVR, self)._estimate_sigma(data)
        self._feature_gen._sigma = self._sigma
        self._feature_gen._gamma = 1.0 / (2.0 * np.square(self._sigma))

    def _source_features(self):
        # the constructor's fit is the first outer iteration's (same gamma); gamma anneals after it, so later ones fit again
        feats, self._first_features = self._first_features, None
        return feats if feats is not None else self._feature_gen.compute(self._source)


def registration_gmmreg(source, target, tf_type_name="rigid", callbacks=[], **kargs):
    """GMMReg of source to target; tf_type_name 'rigid' or 'nonrigid' (TPS); callbacks get the transformation at every BFGS
    iteration; keyword args go to RigidGMMReg / TPSGMMReg.  Returns the transformation from source to target."""
    cv = lambda x: np.asarray(x.points if hasattr(x, "points") else x)  # noqa: E731 (open3d clouds pass their points)
    if tf_type_name == "rigid":
        gmmreg = RigidGMMReg(cv(source), **kargs)
    elif tf_type_name == "nonrigid":
        gmmreg = TPSGMMReg(cv(source), **kargs)
    else:
        raise ValueError("Unknown transform type %s" % tf_type_name)
    gmmreg.set_callbacks(callbacks)
    return gmmreg.registration(cv(target))


def registration_svr(source, target, tf_type_name="rigid", maxiter=1, tol=1.0e-3, opt_maxiter=50, opt_tol=1.0e-3, callbacks=[],
                     **kwargs):
    """Support vector registration of source to target; tf_type_name 'rigid' or 'nonrigid' (TPS); maxiter / tol: the outer loop,
    opt_maxiter / opt_tol: BFGS; callbacks get the transformation at every BFGS iteration; keyword args go to RigidSVR / TPSSVR.
    Returns the transformation from source to target."""
    cv = lambda x: np.asarray(x.points if hasattr(x, "points") else x)  # noqa: E731 (open3d clouds pass their points)
    if tf_type_name == "rigid":
        svr = RigidSVR(cv(source), **kwargs)
    elif tf_type_name == "nonrigid":
        svr = TPSSVR(cv(source), **kwargs)
    else:
        raise ValueError("Unknown transform type %s" % tf_type_name)
    svr.set_callbacks(callbacks)
    return svr.registration(cv(target), maxiter, tol, opt_maxiter, opt_tol)
