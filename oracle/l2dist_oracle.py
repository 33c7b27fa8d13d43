"""Float64 numpy restatement of GMMReg (probreg/l2dist_regs.py, cost_functions.py, features.py, se3_op.py, transformation.py,
cc/math_utils.cc) -- the oracle the tests compare cpd_gmm_fit, cpd_l2_dist, cpd_tps_kernel and probreg_b200.l2dist_regs against.

  * gmm_fit: sklearn's GaussianMixture(covariance_type="spherical", init_params="random_from_data", n_init=1).fit, with
    sklearn's own formulas (sklearn/mixture/_gaussian_mixture.py: _estimate_gaussian_parameters with the avg_X2 - 2 avg_X_means +
    avg_means2 expansion of _estimate_gaussian_covariances_spherical, _estimate_log_gaussian_prob's expanded log-probabilities;
    _base.py: _initialize, fit_predict's E-step / M-step / stop-test order), over the points in chunks so that 100k x 800 fits
    in memory;
  * l2_dist: compute_l2_dist (cost_functions.py:33-41) with the Gauss transforms as direct float64 sums (the reference's
    GaussTransform is an IFGT);
  * quat2mat (transforms3d's formula), diff_rot_from_quaternion (se3_op.py:62-…, its values, see below), tps_kernel
    (cc/math_utils.cc:21-30, float32), TPS prepare (transformation.py:141-156), the rigid and TPS cost functions
    (cost_functions.py:44-112) and the BFGS outer loop (l2dist_regs.py:71-97).
"""
import numpy as np
from scipy.optimize import minimize
from scipy.special import logsumexp

EPS = np.finfo(np.float64).eps
CHUNK = 8192


# ---- the spherical GMM fit ---------------------------------------------------------------------------------------------------------
def _moments(X, means, var, w, chunk=CHUNK):
    """one E-step over X in chunks: (mean lse, sum resp, resp^T X, resp^T X^2)"""
    n, d = X.shape
    prec_chol = 1.0 / np.sqrt(var)
    log_det = d * np.log(prec_chol)
    prec = prec_chol ** 2
    m2 = np.sum(means ** 2, 1) * prec
    k = len(w)
    s0, s1, s2, lse_sum = np.zeros(k), np.zeros((k, d)), np.zeros((k, d)), 0.0
    for a in range(0, n, chunk):
        x = X[a:a + chunk]
        log_prob = m2 - 2.0 * np.dot(x, means.T * prec) + np.outer(np.sum(x * x, 1), prec)
        wlp = -0.5 * (d * np.log(2.0 * np.pi) + log_prob) + log_det + np.log(w)
        lse = logsumexp(wlp, axis=1)
        resp = np.exp(wlp - lse[:, None])
        s0 += resp.sum(0)
        s1 += resp.T.dot(x)
        s2 += resp.T.dot(x * x)
        lse_sum += lse.sum()
    return lse_sum / n, s0, s1, s2


def _params(s0, s1, s2, reg):
    """_estimate_gaussian_parameters + _estimate_gaussian_covariances_spherical from the sums"""
    nk = s0 + 10.0 * EPS
    means = s1 / nk[:, None]
    avg_x2 = s2 / nk[:, None]
    avg_x_means = means * s1 / nk[:, None]
    var = (avg_x2 - 2.0 * avg_x_means + means ** 2 + reg).mean(1)
    return nk, means, var


def random_from_data(n, k, seed):
    return np.random.RandomState(seed).choice(n, k, replace=False)


def gmm_fit(X, k, seed=0, seeds=None, reg_covar=1e-6, tol=1e-3, max_iter=100, chunk=CHUNK):
    """(weights, means, variances, n_iter, lower bound per iteration)"""
    X = np.asarray(X, dtype=np.float64)
    n = len(X)
    idx = random_from_data(n, k, seed) if seeds is None else np.asarray(seeds)
    s0 = np.ones(k)                                     # one-hot responsibilities at the seeds (_base.py _initialize)
    s1 = X[idx].copy()
    s2 = X[idx] ** 2
    nk, means, var = _params(s0, s1, s2, reg_covar)
    w = nk / n                                          # not normalised: sklearn's _initialize divides by n_samples
    lb, lbs = -np.inf, []
    for it in range(1, max_iter + 1):
        prev = lb
        lb, s0, s1, s2 = _moments(X, means, var, w, chunk)
        nk, means, var = _params(s0, s1, s2, reg_covar)
        w = nk / nk.sum()
        lbs.append(lb)
        if abs(lb - prev) < tol:
            break
    return w, means, var, it, np.array(lbs)


# ---- the L2 distance ---------------------------------------------------------------------------------------------------------------
def gauss_transform(src, tgt, h, weights, chunk=2048):
    """out[..., i] = sum_j weights[..., j] exp(-|src_i - tgt_j|^2 / h^2), direct"""
    weights = np.atleast_2d(weights)
    out = np.zeros((weights.shape[0], len(src)))
    for a in range(0, len(src), chunk):
        d2 = ((src[a:a + chunk, None, :] - tgt[None, :, :]) ** 2).sum(-1)
        out[:, a:a + chunk] = weights.dot(np.exp(-d2 / (h * h)).T)
    return out


def l2_dist(mu_source, phi_source, mu_target, phi_target, sigma):
    """cost_functions.py:33-41"""
    z = np.power(2.0 * np.pi * sigma ** 2, mu_source.shape[1] * 0.5)
    h = np.sqrt(2.0) * sigma
    phi_j_e = gauss_transform(mu_source, mu_target, h, phi_target / z)[0]
    phi_mu_j_e = gauss_transform(mu_source, mu_target, h, phi_target * mu_target.T / z).T
    g = (phi_source * phi_j_e * mu_source.T - phi_source * phi_mu_j_e.T).T / (2.0 * sigma ** 2)
    return -np.dot(phi_source, phi_j_e), g


# ---- rotations ---------------------------------------------------------------------------------------------------------------------
def _amat(q):
    w, x, y, z = q
    return np.array([[-(y * y + z * z), x * y - w * z, x * z + w * y], [x * y + w * z, -(x * x + z * z), y * z - w * x],
                     [x * z - w * y, y * z + w * x, -(x * x + y * y)]])


def quat2mat(q):
    """transforms3d.quaternions.quat2mat: I + 2 A(q) / |q|^2"""
    n = float(np.dot(q, q))
    if n < EPS:
        return np.identity(3)
    return np.identity(3) + 2.0 / n * _amat(q)


def diff_rot_from_quaternion(q):
    """The values of se3_op.py:62-…: the quotient rule of R = I + 2 A / N (A quadratic, so its central difference with step 1 is
    its exact derivative), with the reference's two departures from the exact derivative: the off-diagonal normalisation term is
    2 q_k R / N^2 (exact: / N), and dR_22/dq_2, dR_22/dq_3 carry the factors (q_1^2 + q_2^2), (q_3^2 + q_0^2) (se3_op.py, the
    d_rot[2, 2, 2] and d_rot[3, 2, 2] lines)."""
    q = np.asarray(q, dtype=np.float64)
    n = float(np.dot(q, q))
    rot = quat2mat(q)
    a = _amat(q)
    d = np.zeros((4, 3, 3))
    for k in range(4):
        e = np.zeros(4)
        e[k] = 1.0
        da = 0.5 * (_amat(q + e) - _amat(q - e))
        d[k] = 2.0 / n * da
        for i in range(3):
            for j in range(3):
                d[k, i, j] -= 4.0 * q[k] * a[i, i] / n ** 2 if i == j else 2.0 * q[k] * rot[i, j] / n ** 2
    q2 = q * q
    d[2, 2, 2] = -4.0 * q[2] * (q2[1] + q2[2]) / n ** 2
    d[3, 2, 2] = 4.0 * q[3] * (q2[3] + q2[0]) / n ** 2
    return d


# ---- TPS ---------------------------------------------------------------------------------------------------------------------------
def tps_kernel(x, y):
    """cc/math_utils.cc:21-30 in float32, every operation rounded on its own: 2-D r^2 log r (0 where r^2 <= 1e-9; the log of the
    float32 r in float64, rounded once), 3-D -r"""
    x32, y32 = np.asarray(x, dtype=np.float32), np.asarray(y, dtype=np.float32)
    dim = x32.shape[1]
    d2 = np.zeros((len(x32), len(y32)), dtype=np.float32)
    for a in range(dim):
        dd = x32[:, None, a] - y32[None, :, a]
        d2 = d2 + dd * dd
    r = np.sqrt(d2)
    if dim == 2:
        with np.errstate(divide="ignore", invalid="ignore"):
            lg = np.log(r.astype(np.float64)).astype(np.float32)
            return np.where(d2 > np.float32(1e-9), d2 * lg, np.float32(0.0)).astype(np.float32)
    return (-r).astype(np.float32)


def tps_prepare(landmarks, control_pts):
    """transformation.py:141-153: (basis, kernel)"""
    m, d = landmarks.shape
    n = control_pts.shape[0]
    pm = np.c_[np.ones((m, 1)), landmarks]
    pn = np.c_[np.ones((n, 1)), control_pts]
    u, _, _ = np.linalg.svd(pn)
    pp = u[:, d + 1:]
    basis = np.c_[pm, np.dot(tps_kernel(landmarks, control_pts), pp)]
    return basis, np.dot(pp.T, np.dot(tps_kernel(control_pts, control_pts), pp))


# ---- cost functions and the outer loop ---------------------------------------------------------------------------------------------
def rigid_cost(theta, mu_source, phi_source, mu_target, phi_target, sigma):
    """RigidCostFunction.__call__ (cost_functions.py:60-68)"""
    rot = quat2mat(theta[:4])
    f, g = l2_dist(mu_source.dot(rot.T) + theta[4:7], phi_source, mu_target, phi_target, sigma)
    gtm0 = g.T.dot(mu_source)
    return f, np.concatenate([(gtm0 * diff_rot_from_quaternion(theta[:4])).sum(axis=(1, 2)), g.sum(axis=0)])


class TPSCost(object):
    """TPSCostFunction (cost_functions.py:71-112) with the basis of one source mixture"""

    def __init__(self, control_pts, alpha=1.0, beta=0.1):
        self.ctrl, self.alpha, self.beta = control_pts, alpha, beta
        self._prep = None

    def split(self, theta):
        dim = self.ctrl.shape[1]
        n_a = dim * (dim + 1)
        return theta[:n_a].reshape(dim + 1, dim), theta[n_a:].reshape(-1, dim)

    def initial(self):
        dim = self.ctrl.shape[1]
        return np.r_[np.zeros((1, dim)), np.identity(dim), np.zeros((self.ctrl.shape[0] - dim - 1, dim))].flatten()

    def __call__(self, theta, mu_source, phi_source, mu_target, phi_target, sigma):
        dim = self.ctrl.shape[1]
        if self._prep is None or self._prep[0] is not mu_source:
            self._prep = (mu_source,) + tps_prepare(mu_source, self.ctrl)
        basis, kernel = self._prep[1:]
        a, v = self.split(theta)
        t_mu = basis.dot(np.r_[a, v])
        bending = np.trace(v.T.dot(kernel.dot(v)))
        f1, g1 = l2_dist(t_mu, phi_source, t_mu, phi_source, sigma)
        f2, g2 = l2_dist(t_mu, phi_source, mu_target, phi_target, sigma)
        grad = self.alpha * basis.T.dot(-2.0 * g1 + 2.0 * g2)
        grad[dim + 1:, :] += 2.0 * self.beta * kernel.dot(v)
        return self.alpha * (-f1 + 2.0 * f2) + self.beta * bending, grad.flatten()


def estimate_sigma(data):
    """l2dist_regs.py:61-64"""
    data_hat = data - data.mean(0)
    return np.power(np.linalg.det(data_hat.T.dot(data_hat) / (len(data) - 1)), 1.0 / (2.0 * data.shape[1]))


def registration(cost, x0, features_src, features_tgt, sigma, delta=0.9, maxiter=1, tol=1e-3, opt_maxiter=50, opt_tol=1e-3):
    """l2dist_regs.py:71-97 with fixed features per outer iteration; returns the final theta"""
    f, x_ini = None, x0
    for _ in range(maxiter):
        res = minimize(cost, x_ini, args=features_src + features_tgt + (sigma,), method="BFGS", jac=True, tol=opt_tol,
                       options={"maxiter": opt_maxiter})
        sigma *= delta
        if f is not None and abs(res.fun - f) < tol:
            break
        f, x_ini = res.fun, res.x
    return res.x
