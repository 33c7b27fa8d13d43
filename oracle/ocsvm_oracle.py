"""Float64 oracle of the one-class SVM fit behind probreg's SVR features (features.OneClassSVM: sklearn's
``OneClassSVM(kernel="rbf", nu, gamma).fit``), restated from the published algorithm: libsvm's SMO with second-order working-set
selection (Fan, Chen & Lin, JMLR 2005), without shrinking, run the way sklearn runs it.

The dual: min 1/2 a^T Q a subject to 0 <= a_i <= 1 and sum a = nu l, with Q_ij = exp(-gamma |x_i - x_j|^2).  For smooth kernels it
is badly conditioned, so a solution to the same tolerance by another path has different support vectors and weights; these
details make the path sklearn's own:
  * start: nu_l accumulated serially (l additions of nu), then a_i = min(1, nu_l), nu_l -= a_i, i = 0, 1, ... while nu_l > 0
    (sklearn's sample-weighted start; its float residue leaves a tiny extra a);
  * kernel: exp(-gamma (|x_i|^2 + |x_j|^2 - 2 x_i.x_j)) on the raw coordinates, dot products summed over the dimensions in order,
    rounded to float32 (libsvm's Qfloat column cache) and used as a double afterwards; Q_ii = 1 exactly;
  * selection: i = argmax of -G over a < 1, j = argmin of -(Gmax + G_t)^2 / (2 - 2 Q_it) over a > 0 with Gmax + G_t > 0 (a quad
    <= 0 becomes 1e-12); ties to the largest index (libsvm's >= / <= scans); stop when Gmax + max_{a>0} G < tol or there is no j;
  * update: libsvm's clipped two-variable step for equal labels, then G += Q_i da_i + Q_j da_j (the two products added first);
    the start's G = sum_i a_i Q_i accumulated over i in increasing order;
  * rho: the mean of G over the free a; with none, the midpoint of min G over a = 0 and max G over a = 1.  sklearn reports
    intercept_ = -rho.
n_iter counts the updates (0 when nu = 1).  O(l) work per iteration, vectorised.
"""
import numpy as np

TAU = 1e-12


def default_max_iter(n):
    """libsvm's cap when sklearn passes max_iter = -1"""
    return max(10_000_000, 100 * n)


def _sq(x):
    s = np.zeros(len(x))
    for c in range(x.shape[1]):
        s = s + x[:, c] * x[:, c]
    return s


def kernel_column(x, xsq, i, gamma):
    dot = np.zeros(len(x))
    for c in range(x.shape[1]):
        dot = dot + x[:, c] * x[i, c]
    return np.exp(-gamma * (xsq[i] + xsq - 2.0 * dot)).astype(np.float32).astype(np.float64)


def start_alpha(n, nu):
    a = np.zeros(n)
    nul = 0.0
    for _ in range(n):
        nul += 1.0 * nu
    k = 0
    while nul > 0 and k < n:
        a[k] = min(1.0, nul)
        nul -= a[k]
        k += 1
    return a


def rho(a, G):
    free = (a > 0.0) & (a < 1.0)
    if free.any():
        return G[free].sum() / free.sum()
    ub = G[a <= 0.0].min() if (a <= 0.0).any() else np.inf
    lb = G[a >= 1.0].max() if (a >= 1.0).any() else -np.inf
    return (ub + lb) / 2.0


def fit(x, nu, gamma, tol=1e-3, max_iter=None):
    """(alpha (all l points), rho, n_iter, G)"""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    max_iter = default_max_iter(n) if max_iter is None else max_iter
    xsq = _sq(x)
    a = start_alpha(n, nu)
    G = np.zeros(n)
    for i in np.nonzero(a)[0]:
        G += a[i] * kernel_column(x, xsq, i, gamma)
    it = 0
    while it < max_iter:
        mg = np.where(a < 1.0, -G, -np.inf)
        i = n - 1 - np.argmax(mg[::-1])
        gmax = mg[i]
        lo = a > 0.0
        gmax2 = np.max(np.where(lo, G, -np.inf))
        gd = gmax + G
        if np.isfinite(gmax):
            Qi = kernel_column(x, xsq, i, gamma)
            quad = 1.0 + 1.0 - 2.0 * Qi
            quad = np.where(quad <= 0.0, TAU, quad)
            od = np.where(lo & (gd > 0.0), -(gd * gd) / quad, np.inf)
        else:
            od = np.full(n, np.inf)
        if gmax + gmax2 < tol or not np.isfinite(od.min()):
            break
        j = n - 1 - np.argmin(od[::-1])
        Qj = kernel_column(x, xsq, j, gamma)
        ai, aj = a[i], a[j]
        qc = 1.0 + 1.0 - 2.0 * Qi[j]
        if qc <= 0.0:
            qc = TAU
        delta = (G[i] - G[j]) / qc
        s = ai + aj
        a[i] -= delta
        a[j] += delta
        if s > 1.0:
            if a[i] > 1.0:
                a[i], a[j] = 1.0, s - 1.0
        elif a[j] < 0.0:
            a[j], a[i] = 0.0, s
        if s > 1.0:
            if a[j] > 1.0:
                a[j], a[i] = 1.0, s - 1.0
        elif a[i] < 0.0:
            a[i], a[j] = 0.0, s
        G += Qi * (a[i] - ai) + Qj * (a[j] - aj)
        it += 1
    return a, rho(a, G), it, G


def svr_features(x, sigma, gamma, nu, tol=1e-3):
    """features.OneClassSVM.compute: (support vectors, alpha_sv (2 pi sigma^2)^(D/2))"""
    a = fit(x, nu, gamma, tol)[0]
    sv = a > 0.0
    return x[sv], a[sv] * np.power(2.0 * np.pi * sigma ** 2, x.shape[1] * 0.5)


def registration(cost, x0, source, target, sigma, gamma, nu=0.1, delta=0.9, gamma_delta=10.0, maxiter=1, tol=1e-3,
                 opt_maxiter=50, opt_tol=1e-3, features=None):
    """l2dist_regs.py:71-97 for RigidSVR / TPSSVR: per outer iteration both clouds' features at the current gamma (features(data,
    gamma), svr_features by default), a BFGS solve from the last solution, then sigma *= delta and gamma *= gamma_delta (the
    feature's sigma stays the estimated one).  Returns the final theta."""
    from scipy.optimize import minimize

    feat_sigma = sigma
    features = features or (lambda d, g: svr_features(d, feat_sigma, g, nu))
    f, x_ini = None, x0
    for _ in range(maxiter):
        ms, ps = features(source, gamma)
        mt, pt = features(target, gamma)
        res = minimize(cost, x_ini, args=(ms, ps, mt, pt, sigma), method="BFGS", jac=True, tol=opt_tol, options={"maxiter": opt_maxiter})
        sigma *= delta
        gamma *= gamma_delta
        if f is not None and abs(res.fun - f) < tol:
            break
        f, x_ini = res.fun, res.x
    return res.x
