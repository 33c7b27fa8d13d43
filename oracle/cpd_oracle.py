"""CPU oracle for the CPD EM hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

This module is a numpy/scipy restatement of the algorithm that neka-nat/probreg
(v0.3.7) runs on its numpy path.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s CPU-baseline / ``--impl reference`` legs may import it, and only as
the checker or the CPU arm being timed.  Nothing under ``probreg_b200/`` imports it;
the product path has no CPU fallback.

Parity status: PINNED.  ``tests/golden/make_golden.py`` imports the reference's own
``probreg/cpd.py`` unmodified (from a reference checkout named by $PROBREG_REFERENCE)
and stores its outputs in ``tests/golden/*.npz``; ``tests/test_oracle.py``
checks every function below against those fixtures.

Reference lines restated here (all paths relative to the reference repo):

* sigma^2 initialisation   probreg/math_utils.py:28-29 -> probreg/cc/math_utils.cc:5-15
                           (float32 Eigen matrix, probreg/cc/types.h:19)
* RBF Gram matrix          probreg/math_utils.py:36-37 -> probreg/cc/math_utils.cc:17-19
* E-step                   probreg/cpd.py:71-88
* rigid M-step             probreg/cpd.py:160-192
* affine M-step            probreg/cpd.py:219-244
* non-rigid M-step         probreg/cpd.py:284-303
* transforms               probreg/transformation.py:49-50, 77-78, 101-102
* EM driver                probreg/cpd.py:106-120 (+ _initialize :145-153 / :209-217 / :277-282)

The one structural difference from the reference: the E-step walks the target
columns in blocks so that the M x N matrix never has to exist at once (the
reference needs 24*M*N bytes, i.e. 240 GB at 100k x 100k).  Every quantity of the
E-step is separable per target column, so blocking is exact for ``pt1`` and changes
``p1``/``px`` only by the order of a float64 summation (~1e-15 relative).
"""
from collections import namedtuple

import numpy as np
from scipy.spatial.distance import cdist

EPS32 = float(np.finfo(np.float32).eps)

Estep = namedtuple("Estep", ["pt1", "p1", "px", "n_p"])
Mstep = namedtuple("Mstep", ["params", "sigma2", "q"])


# ---------------------------------------------------------------------------
# probreg._math restated (float32, as the pybind11/Eigen module computes it)
# ---------------------------------------------------------------------------
def squared_kernel_f32(x, y):
    """probreg/cc/math_utils.cc:5-15 -- k[i, j] = |x_i - y_j|^2 in float32.

    The Eigen matrix is column-major; the result is returned Fortran-ordered so
    that a following ``.sum()`` walks memory the way numpy would on the real module.
    """
    xf = np.asarray(x, dtype=np.float32)
    yf = np.asarray(y, dtype=np.float32)
    k = np.empty((xf.shape[0], yf.shape[0]), dtype=np.float32, order="F")
    for j in range(yf.shape[0]):
        d = xf - yf[j]
        acc = d[:, 0] * d[:, 0]
        for a in range(1, xf.shape[1]):
            acc = acc + d[:, a] * d[:, a]
        k[:, j] = acc
    return k


def rbf_kernel_f32(x, y, beta):
    """probreg/cc/math_utils.cc:17-19 -- exp(-|x_i - y_j|^2 / (2*beta)), float32.

    Note the denominator is 2*beta, not 2*beta^2.
    """
    k = squared_kernel_f32(x, y)
    return np.exp(-k / np.float32(2.0 * beta)).astype(np.float32)


def imq_kernel_f32(x, y, c=1.0):
    """probreg/cc/math_utils.cc:37-39 -- (|x_i - y_j|^2 + c)^(-1/2) in float32, every operation rounded on its own
    (squares summed coordinate by coordinate, like Eigen's squaredNorm without FMA contraction)."""
    x32, y32 = np.asarray(x, dtype=np.float32), np.asarray(y, dtype=np.float32)
    d = x32[:, None, :] - y32[None, :, :]
    acc = d[:, :, 0] * d[:, :, 0]
    for a in range(1, x32.shape[1]):
        acc = acc + d[:, :, a] * d[:, :, a]
    return (np.float32(1.0) / np.sqrt(acc + np.float32(c))).astype(np.float32)


def sigma2_init(source, target, max_dense=int(4e7)):
    """probreg/math_utils.py:28-29: mean squared pair distance / D, in float32.

    Dense float32 emulation while M*N <= max_dense; above that the float32 pair
    terms are summed block-wise in float64 (the dense float32 matrix would not fit).
    Returns numpy.float32 like the reference: under numpy>=2 (NEP 50) that dtype
    survives ``2.0 * sigma2`` and the outlier constant of the FIRST E-step, which are
    therefore evaluated in float32 there (a ~1e-8 relative quirk that the oracle keeps).
    """
    m, d = source.shape
    n = target.shape[0]
    if m * n <= max_dense:
        return squared_kernel_f32(source, target).sum() / (m * d * n)
    xf = np.asarray(source, dtype=np.float32)
    yf = np.asarray(target, dtype=np.float32)
    step = max(1, max_dense // m)
    tot = 0.0
    for j0 in range(0, n, step):
        blk = cdist(xf, yf[j0:j0 + step], "sqeuclidean")
        tot += float(blk.sum())
    return np.float32(tot / (m * d * n))


def sigma2_init_exact(source, target):
    """Closed form of the same quantity in float64."""
    m, d = source.shape
    n = target.shape[0]
    sx = np.sum(target * target)
    sy = np.sum(source * source)
    return float((m * sx + n * sy - 2.0 * target.sum(0).dot(source.sum(0))) / (m * n * d))


# ---------------------------------------------------------------------------
# E-step  (probreg/cpd.py:71-88)
# ---------------------------------------------------------------------------
def outlier_constant(sigma2, w, m, n, dim):
    """cpd.py:78-79 -- uniform-outlier term added to every column sum."""
    c = (2.0 * np.pi * sigma2) ** (dim * 0.5)
    c = c * (w / (1.0 - w) * m / n)
    return c


def expectation_step(t_source, target, sigma2, w=0.0, block=None, n_global=None):
    """Responsibilities and their reductions, never holding more than M x block pairs.

    ``n_global`` is the N that enters the outlier constant (cpd.py:79 uses
    ``target.shape[0]``); pass it when ``target`` is only a shard of the cloud.
    """
    assert t_source.ndim == 2 and target.ndim == 2
    m, dim = t_source.shape
    n = target.shape[0]
    if n_global is None:
        n_global = n
    if block is None:
        block = n if m * n <= int(3e7) else max(1, int(3e7) // m)
    c = outlier_constant(sigma2, w, m, n_global, dim)
    pt1 = np.empty(n)
    p1 = np.zeros(m)
    px = np.zeros((m, dim))
    for j0 in range(0, n, block):
        xb = target[j0:j0 + block]
        k = cdist(t_source, xb, "sqeuclidean")          # cpd.py:74
        k = np.exp(-k / (2.0 * sigma2))                  # cpd.py:76
        den = k.sum(axis=0)                              # cpd.py:80
        den[den == 0] = EPS32                            # cpd.py:81
        den += c                                         # cpd.py:82
        k = k / den                                      # cpd.py:84
        pt1[j0:j0 + block] = k.sum(axis=0)               # cpd.py:85
        p1 += k.sum(axis=1)                              # cpd.py:86
        px += k.dot(xb)                                  # cpd.py:87
    return Estep(pt1, p1, px, float(np.sum(p1)))


# ---------------------------------------------------------------------------
# M-steps
# ---------------------------------------------------------------------------
def _weighted_frames(source, target, es):
    pt1, p1, px, n_p = es
    mu_x = px.sum(axis=0) / n_p                          # cpd.py:171 / :229
    mu_y = source.T.dot(p1) / n_p                        # cpd.py:172 / :230
    xh = target - mu_x
    yh = source - mu_y
    a = px.T.dot(yh) - np.outer(mu_x, p1.dot(yh))        # cpd.py:175 / :233
    return mu_x, mu_y, xh, yh, a


def mstep_rigid(source, target, es, update_scale=True):
    """probreg/cpd.py:160-192.  Returns Mstep((rot, t, scale), sigma2, q)."""
    pt1, p1, px, n_p = es
    dim = source.shape[1]
    mu_x, mu_y, xh, yh, a = _weighted_frames(source, target, es)
    u, _, vh = np.linalg.svd(a, full_matrices=True)      # cpd.py:176
    fix = np.ones(dim)
    fix[-1] = np.linalg.det(u.dot(vh))                   # cpd.py:177-178
    rot = (u * fix).dot(vh)                              # cpd.py:179
    tr_atr = np.trace(a.T.dot(rot))                      # cpd.py:180
    tr_yp1y = np.trace((yh.T * p1).dot(yh))              # cpd.py:181
    scale = tr_atr / tr_yp1y if update_scale else 1.0    # cpd.py:182
    t = mu_x - scale * rot.dot(mu_y)                     # cpd.py:183
    tr_xp1x = np.trace((xh.T * pt1).dot(xh))             # cpd.py:184
    if update_scale:
        sigma2 = (tr_xp1x - scale * tr_atr) / (n_p * dim)            # cpd.py:186
    else:
        sigma2 = (tr_xp1x + tr_yp1y - scale * tr_atr) / (n_p * dim)  # cpd.py:188
    sigma2 = max(sigma2, EPS32)                          # cpd.py:189
    q = (tr_xp1x - 2.0 * scale * tr_atr + scale * scale * tr_yp1y) / (2.0 * sigma2)
    q += dim * n_p * 0.5 * np.log(sigma2)                # cpd.py:190-191
    return Mstep((rot, t, float(scale)), float(sigma2), float(q))


def mstep_affine(source, target, es):
    """probreg/cpd.py:219-244.  Returns Mstep((b, t), sigma2, q)."""
    pt1, p1, px, n_p = es
    dim = source.shape[1]
    mu_x, mu_y, xh, yh, a = _weighted_frames(source, target, es)
    yp1y = (yh.T * p1).dot(yh)                           # cpd.py:234
    b = np.linalg.solve(yp1y.T, a.T).T                   # cpd.py:235
    t = mu_x - b.dot(mu_y)                               # cpd.py:236
    tr_xp1x = np.trace((xh.T * pt1).dot(xh))             # cpd.py:237
    tr_abt = np.trace(a.dot(b.T))                        # cpd.py:238,240
    sigma2 = max((tr_xp1x - tr_abt) / (n_p * dim), EPS32)
    q = (tr_xp1x - 2.0 * tr_abt + tr_abt) / (2.0 * sigma2) + dim * n_p * 0.5 * np.log(sigma2)
    return Mstep((b, t), float(sigma2), float(q))


def constraint_terms(m, target, idx_source, idx_target):
    """probreg/cpd.py:370-374: the dense M x N indicator matrix of known correspondences,
    reduced the way the reference reduces it (row sums, product with the target)."""
    p_tilde = np.zeros((m, target.shape[0]))
    if idx_source is not None and idx_target is not None:
        p_tilde[idx_source, idx_target] = 1
    return p_tilde.sum(axis=1), p_tilde.dot(target)


def mstep_nonrigid(source, target, es, sigma2_p, g, lmd, alpha=None, p1_tilde=None, px_tilde=None):
    """probreg/cpd.py:284-303; with alpha / p1_tilde / px_tilde the constrained variant cpd.py:376-404.
    ``g`` is the (float32) RBF Gram matrix of the source.

    Returns Mstep((w,), sigma2, q) with q == sigma2 as in the reference (cpd.py:303 / :404).
    """
    pt1, p1, px, n_p = es
    m, dim = source.shape
    lhs = (p1 * g).T + lmd * sigma2_p * np.identity(m)   # cpd.py:296
    rhs = px - (source.T * p1).T
    if alpha is not None:
        lhs = lhs + sigma2_p / alpha * (p1_tilde * g).T  # cpd.py:392-394
        rhs = rhs + sigma2_p / alpha * (px_tilde - (source.T * p1_tilde).T)   # cpd.py:395
    wmat = np.linalg.solve(lhs, rhs)
    t = source + g.dot(wmat)                             # cpd.py:297
    tr_xp1x = np.trace((target.T * pt1).dot(target))
    tr_pxt = np.trace(px.T.dot(t))
    tr_tpt = np.trace((t.T * p1).dot(t))
    sigma2 = (tr_xp1x - 2.0 * tr_pxt + tr_tpt) / (n_p * dim)   # cpd.py:301
    return Mstep((wmat,), float(sigma2), float(sigma2))


def lowrank_factors(source, beta, rank, power_iters=2, seed=0):
    """Rank-``rank`` factorisation G ~= Q Bc Q^T of the RBF Gram matrix by the randomised range finder the product uses
    (probreg_b200/csrc/lowrank.cuh): Q = orth((G)^(power_iters+1) Omega), Bc = Q^T G Q.  No reference counterpart (the
    reference only has the dense G); test infrastructure for the low-rank path.  numpy QR instead of Gram-Schmidt and
    another random Omega, so only quantities that do not depend on the basis (Q Bc Q^T, the moved points, sigma2) are
    comparable with the product."""
    g = rbf_kernel_f32(source, source, beta).astype(np.float64)
    m = source.shape[0]
    rank = min(rank, m)
    x = np.random.default_rng(seed).uniform(-1.0, 1.0, (m, rank))
    for _ in range(power_iters + 1):
        x, _r = np.linalg.qr(g.dot(x))
    gq = g.dot(x)
    bc = x.T.dot(gq)
    return x, 0.5 * (bc + bc.T)


def mstep_nonrigid_lowrank(source, target, es, sigma2_p, q_mat, bcore, lmd, alpha=None, p1_tilde=None, px_tilde=None):
    """The M-step of cpd.py:284-303 (constrained: :376-404) with G = Q Bc Q^T, solved in the K x K form of lowrank.cuh:
    (c I + Bc S) Z = Bc R,  S = Q^T diag(wgt) Q,  R = Q^T F,  W = (F - diag(wgt) Q Z) / c,  T = Y + Q Z."""
    pt1, p1, px, n_p = es
    dim = source.shape[1]
    wgt, f = p1, px - (source.T * p1).T
    if alpha is not None:
        kk = sigma2_p / alpha
        wgt = p1 + kk * p1_tilde
        f = f + kk * (px_tilde - (source.T * p1_tilde).T)
    c = lmd * sigma2_p
    s_mat = (q_mat.T * wgt).dot(q_mat)
    z = np.linalg.solve(c * np.identity(bcore.shape[0]) + bcore.dot(s_mat), bcore.dot(q_mat.T.dot(f)))
    wmat = (f - (q_mat.T * wgt).T.dot(z)) / c
    t = source + q_mat.dot(z)
    tr_xp1x = np.trace((target.T * pt1).dot(target))
    tr_pxt = np.trace(px.T.dot(t))
    tr_tpt = np.trace((t.T * p1).dot(t))
    sigma2 = (tr_xp1x - 2.0 * tr_pxt + tr_tpt) / (n_p * dim)
    return Mstep((wmat, t), float(sigma2), float(sigma2))


BcpdEstep = namedtuple("BcpdEstep", ["nu_d", "nu", "n_p", "px", "x_hat"])


def bcpd_expectation_step(t_source, target, scale, alpha, sigma_mat, sigma2, w=0.0):
    """probreg/bcpd.py:53-72 (BayesianCoherentPointDrift.expectation_step), restated.

    phi_mn = N(x_n; t_m, sigma2 I) * exp(-scale^2 D sigma_mm / (2 sigma2)) * (1 - w) * alpha_m      (bcpd.py:57-63)
    den_n  = w / N + sum_m phi_mn, zero -> float32 eps                                            (bcpd.py:64-65)
    P = phi / den;  nu_d = sum_m P (N);  nu = sum_n P (M);  px = P x (M x D);  x_hat = px / nu      (bcpd.py:66-72)
    ``sigma_mat`` may be the M x M matrix (only its diagonal is read) or the diagonal itself.
    """
    t_source = np.asarray(t_source, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    m, dim = t_source.shape
    n = target.shape[0]
    sdiag = np.asarray(sigma_mat, dtype=np.float64)
    if sdiag.ndim == 2:
        sdiag = np.diag(sdiag)
    d2 = ((t_source[:, None, :] - target[None, :, :]) ** 2).sum(-1)                  # (M, N)
    phi = np.exp(-d2 / (2.0 * sigma2)) / (2.0 * np.pi * sigma2) ** (dim * 0.5)
    phi = phi * (np.exp(-(scale ** 2) / (2.0 * sigma2) * sdiag * dim) * (1.0 - w) * np.asarray(alpha, dtype=np.float64))[:, None]
    den = w / n + phi.sum(axis=0)
    den[den == 0] = EPS32
    p = phi / den
    nu_d = p.sum(axis=0)
    nu = p.sum(axis=1)
    px = p.dot(target)
    with np.errstate(divide="ignore", invalid="ignore"):
        x_hat = px / nu[:, None]
    return BcpdEstep(nu_d, nu, float(nu.sum()), px, x_hat)


# ---------------------------------------------------------------------------
# transforms (probreg/transformation.py)
# ---------------------------------------------------------------------------
def apply_rigid(points, rot, t, scale=1.0):
    return scale * points.dot(rot.T) + t                 # transformation.py:49-50


def apply_affine(points, b, t):
    return points.dot(b.T) + t                           # transformation.py:77-78


def apply_nonrigid(points, g, wmat):
    return points + g.dot(wmat)                          # transformation.py:101-102


# ---------------------------------------------------------------------------
# EM driver (probreg/cpd.py:106-120)
# ---------------------------------------------------------------------------
def registration(source, target, tf_type="rigid", w=0.0, maxiter=50, tol=1e-3,
                 update_scale=True, beta=2.0, lmd=2.0, sigma2_0=None, init=None,
                 block=None, trace=None, alpha=None, idx_source=None, idx_target=None, g=None):
    """Runs the reference's loop.  Returns (Mstep, iterations_run).

    ``sigma2_0`` overrides the float32-emulated initial variance; ``init`` overrides
    the identity start ((rot, t, scale) or (b, t)); ``trace``, if a list, receives
    (sigma2, q) after every iteration; ``g`` replaces the RBF Gram matrix of the non-rigid
    families (used to check the low-rank product path against the reference's dense
    arithmetic on the SAME approximate G = Q Bc Q^T).
    """
    source = np.asarray(source, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    m, dim = source.shape
    n = target.shape[0]
    sigma2 = sigma2_init(source, target) if sigma2_0 is None else sigma2_0
    q = 1.0 + n * dim * 0.5 * np.log(sigma2)             # cpd.py:148
    if tf_type == "rigid":
        params = (np.identity(dim), np.zeros(dim), 1.0) if init is None else init
    elif tf_type == "affine":
        params = (np.identity(dim), np.zeros(dim)) if init is None else init
    elif tf_type in ("nonrigid", "nonrigid_constrained"):
        if g is None:
            g = rbf_kernel_f32(source, source, beta)      # transformation.py:91-99
        params = (np.zeros_like(source),)                 # cpd.py:281
        prior = {}
        if tf_type == "nonrigid_constrained":
            p1t, pxt = constraint_terms(m, target, idx_source, idx_target)
            prior = {"alpha": 1e-8 if alpha is None else alpha, "p1_tilde": p1t, "px_tilde": pxt}
    else:
        raise ValueError("Unknown transformation type %s" % tf_type)
    res = Mstep(params, sigma2, q)
    it = 0
    for it in range(1, maxiter + 1):
        if tf_type == "rigid":
            ts = apply_rigid(source, *res.params)
        elif tf_type == "affine":
            ts = apply_affine(source, *res.params)
        else:
            ts = apply_nonrigid(source, g, res.params[0])
        es = expectation_step(ts, target, res.sigma2, w, block=block)
        if tf_type == "rigid":
            res = mstep_rigid(source, target, es, update_scale)
        elif tf_type == "affine":
            res = mstep_affine(source, target, es)
        else:
            res = mstep_nonrigid(source, target, es, res.sigma2, g, lmd, **prior)
        if trace is not None:
            trace.append((res.sigma2, res.q))
        if abs(res.q - q) < tol:                          # cpd.py:117
            break
        q = res.q
    return res, it


# ---------------------------------------------------------------------------
# synthetic workloads of BASELINE.md section 3 (shared by tests and bench)
# ---------------------------------------------------------------------------
def rot_z(deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def synthetic_pair(n, kind="rigid", noise=0.01, seed=0):
    """source = anisotropic uniform box; target = permuted, noised, transformed copy."""
    src = np.random.default_rng(seed).random((n, 3)) * np.array([1.0, 0.6, 0.3])
    rng1 = np.random.default_rng(seed + 1)
    perm = rng1.permutation(n)
    pts = src[perm] + noise * rng1.standard_normal((n, 3))
    lin = rot_z(30.0)
    if kind == "affine":
        lin = lin.dot(np.diag([1.1, 0.9, 1.05]))
        lin[0, 1] += 0.05
    tgt = pts.dot(lin.T) + np.array([0.1, -0.2, 0.3])
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)
