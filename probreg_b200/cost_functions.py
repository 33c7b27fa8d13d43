"""Cost functions of ``probreg.cost_functions`` (reference: cost_functions.py) with the L2 distance on the H100.

``compute_l2_dist`` is one device call (``cpd_l2_dist``): direct FP64 sums over every (source, target) component pair, the
gradient accumulated in residual form.  The reference forms it from two float32 IFGT Gauss transforms (eps = 1e-4), so it is
approximate there and exact here.  The chain rules (rigid: through the quaternion; TPS: through the spline basis) stay in numpy:
they are O(components).

``TPSCostFunction`` computes the spline basis and kernel of its source (``TPSTransformation.prepare``) once per source mixture and
reuses them while the optimiser varies (a, v): they do not depend on (a, v), so every evaluation gives what the reference's does.
"""
import abc

import numpy as np

from . import _cabi
from . import se3_op as so
from . import transformation as tf


class CostFunction(abc.ABC):
    def __init__(self, tf_type):
        self._tf_type = tf_type

    @abc.abstractmethod
    def to_transformation(self, theta):
        return None

    @abc.abstractmethod
    def initial(self):
        return None

    @abc.abstractmethod
    def __call__(self, theta, *args):
        return None, None


def compute_l2_dist(mu_source, phi_source, mu_target, phi_target, sigma, device=0):
    """(f, g): f = -sum_i phi_s,i sum_j (phi_t,j / z) e_ij, g_i = phi_s,i sum_j (phi_t,j / z) e_ij (mu_s,i - mu_t,j) / (2 sigma^2),
    z = (2 pi sigma^2)^(D/2), e_ij = exp(-|mu_s,i - mu_t,j|^2 / (2 sigma^2))  (cost_functions.py:33-41)."""
    return _cabi.l2_dist(mu_source, phi_source, mu_target, phi_target, sigma, device)


class RigidCostFunction(CostFunction):
    """theta = (quaternion (4), t (3)); f and its gradient of the moved source mixture against the target's."""

    def __init__(self, device=0):
        self._tf_type = tf.RigidTransformation
        self._device = device

    def to_transformation(self, theta):
        rot = so.quat2mat(theta[:4])
        return self._tf_type(rot, theta[4:7])

    def initial(self):
        x0 = np.zeros(7)
        x0[0] = 1.0
        return x0

    def __call__(self, theta, *args):
        mu_source, phi_source, mu_target, phi_target, sigma = args
        tf_obj = self.to_transformation(theta)
        t_mu_source = tf_obj.transform(mu_source)
        f, g = compute_l2_dist(t_mu_source, phi_source, mu_target, phi_target, sigma, self._device)
        d_rot = so.diff_rot_from_quaternion(theta[:4])
        gtm0 = np.dot(g.T, mu_source)
        grad = np.concatenate([(gtm0 * d_rot).sum(axis=(1, 2)), g.sum(axis=0)])
        return f, grad


class TPSCostFunction(CostFunction):
    """theta = (a ((D + 1) x D), v ((n - D - 1) x D)) flattened, n control points; alpha weighs the L2 terms, beta the bending
    energy trace(v^T K v)."""

    def __init__(self, control_pts, alpha=1.0, beta=0.1, device=0):
        self._tf_type = tf.TPSTransformation
        self._alpha = alpha
        self._beta = beta
        self._control_pts = control_pts
        self._device = device
        self._prepared = None                 # (source mixture, control points, basis, kernel)

    def to_transformation(self, theta):
        dim = self._control_pts.shape[1]
        n_data = theta.shape[0] // dim
        n_a = dim * (dim + 1)
        a = theta[:n_a].reshape(dim + 1, dim)
        v = theta[n_a:].reshape(n_data - dim - 1, dim)
        return self._tf_type(a, v, self._control_pts)

    def initial(self):
        dim = self._control_pts.shape[1]
        a = np.r_[np.zeros((1, dim)), np.identity(dim)]
        v = np.zeros((self._control_pts.shape[0] - dim - 1, dim))
        return np.r_[a, v].flatten()

    def _prepare(self, tf_obj, mu_source):
        p = self._prepared
        if p is None or p[0] is not mu_source or p[1] is not self._control_pts:
            p = self._prepared = (mu_source, self._control_pts) + tf_obj.prepare(mu_source)
        return p[2], p[3]

    def __call__(self, theta, *args):
        dim = self._control_pts.shape[1]
        mu_source, phi_source, mu_target, phi_target, sigma = args
        tf_obj = self.to_transformation(theta)
        basis, kernel = self._prepare(tf_obj, mu_source)
        t_mu_source = tf_obj.transform_basis(basis)
        bending = np.trace(np.dot(tf_obj.v.T, np.dot(kernel, tf_obj.v)))
        f1, g1 = compute_l2_dist(t_mu_source, phi_source, t_mu_source, phi_source, sigma, self._device)
        f2, g2 = compute_l2_dist(t_mu_source, phi_source, mu_target, phi_target, sigma, self._device)
        f = -f1 + 2.0 * f2
        g = -2.0 * g1 + 2.0 * g2
        grad = self._alpha * np.dot(basis.T, g)
        grad[dim + 1:, :] += 2.0 * self._beta * np.dot(kernel, tf_obj.v)
        return self._alpha * f + self._beta * bending, grad.flatten()
