"""Low-rank BCPD (cpd_bcpd_lowrank_begin, CombinedBCPD(low_rank=K)): the loop with G ~= Q Bc Q^T of the inverse multiquadric.

  1. the device loop against a numpy restatement of the low-rank M-step on the SAME exported factors (written with eigh of Bc,
     not with the device's Cholesky factor), after the library's weighted E-step, iteration by iteration;
  2. at K = M on clouds whose G^-1 is well conditioned, the dense loop fed the float32 inverse;
  3. the IMQ G X products element by element against float64, within a bound derived from the arithmetic;
  4. the quality of the factors on boxes of extent 1 and 3;
  5. a cloud of extent 0.5, where the dense loop fails and the low-rank one does not;
  6. the refusals and the interplay of the low-rank factors shared with non-rigid CPD;
  7. (GPU) 100 000 points at K = 200 within 2 GB of device memory, reproducibly;
  8. the Python surface.
CPU tests run under the emulation of tests/emu (M <= 500, CUDA-core products only); the gpu-marked ones on the H100.
"""
import math

import numpy as np
import pytest
from scipy.special import digamma

from probreg_b200 import _cabi, bcpd, math_utils
from probreg_b200 import transformation as tf
from test_zz_bcpd_loop import CASES, _device_loop, _gmat_inv, _pair, _targets

TC, CC = _cabi.Handle.GRAM_TENSOR_CORES, _cabi.Handle.GRAM_CUDA_CORES
U = 2.0 ** -24                     # unit round-off of float32
# 1e-6: see _check_vs_oracle
TOL = 1e-6


def _box_pair(m, dim, extent, seed, far=False):
    """_pair's source and target scaled so that the source spans `extent` (in units of sqrt(c), c = 1)."""
    src, tgt = _pair(m, dim, seed)
    f = extent / np.ptp(src, axis=0).max()
    src, tgt = src * f, tgt * f
    if far:
        src[-1] = 100.0 * extent
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)


def _imq64(a, b, c=1.0):
    d2 = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    return 1.0 / np.sqrt(d2 + c)


# ---- 1. the loop against an oracle on the same factors ---------------------------------------------------------------------------
def _oracle_mstep(src, tgt, trans, es, q, bc, lmd, k, sigma2_p):
    """The low-rank M-step in numpy: G ~= Qt' Qt'^T with Qt' = Q U diag(sqrt(lambda)) from eigh(Bc) (a rotation of the device's
    Qt = Q L, which the algebra does not see); C = (c I + Qt'^T N Qt')^-1, c = lmd / ratio; v = Qt' C Qt'^T r;
    diag Sigma = diag(Qt' C Qt'^T) / ratio; then the dense M-step's mixing weights, similarity and sigma2."""
    nu_d, nu, n_p, px, x_hat = es
    rig = trans.rigid_trans
    ratio = (rig.scale / sigma2_p) ** 2
    lam, vec = np.linalg.eigh(bc)
    qt = q.dot(vec * np.sqrt(np.clip(lam, 0.0, None)))
    c = lmd / ratio
    cmat = np.linalg.inv(c * np.identity(len(lam)) + qt.T.dot(nu[:, None] * qt))
    resid = (px - nu[:, None] * rig.t).dot(rig.rot) / rig.scale - nu[:, None] * src        # R^T (px - nu t) / s - nu y
    v = qt.dot(cmat.dot(qt.T.dot(resid)))
    sdiag = np.einsum("ik,kl,il->i", qt, cmat, qt) / ratio
    u_hat = src + v
    alpha = np.exp(digamma(k + nu) - digamma(k * src.shape[0] + n_p))
    var_term = nu.dot(sdiag) / n_p
    rot, scale, t = bcpd._similarity_from_moments(nu, n_p, x_hat, u_hat, var_term)
    sigma2 = bcpd._residual_variance(tgt, nu_d, nu, n_p, px, rig.transform(u_hat), scale, var_term)
    return tf.CombinedTransformation(rot, t, scale, v), alpha, sdiag, sigma2


def _oracle_loop(src, tgt, q, bc, lmd, k, w, sigma2, iters):
    """[(rot, t, scale, v, sigma2, alpha, sigma_diag)]: library E-step (on a handle holding the ORIGINAL source, like the device
    loop) + _oracle_mstep"""
    dim = src.shape[1]
    h = _cabi.Handle(dim)
    h.set_source(src)
    trans = tf.CombinedTransformation(np.identity(dim), np.zeros(dim))
    alpha, sdiag = np.full(src.shape[0], 1.0 / src.shape[0]), np.ones(src.shape[0])
    out, last = [], None
    for tg in _targets(tgt, iters):
        if tg is not last:
            h.set_target(tg)
            last = tg
        nu_d, nu, px, n_p = h.bcpd_estep(trans.transform(src), trans.rigid_trans.scale, alpha, sdiag, sigma2, w)
        with np.errstate(divide="ignore", invalid="ignore"):
            x_hat = np.where(nu[:, None] > 0, px / nu[:, None], 0.0)
        trans, alpha, sdiag, sigma2 = _oracle_mstep(src, tg, trans, bcpd.EstepResult(nu_d, nu, n_p, px, x_hat), q, bc, lmd, k, sigma2)
        r = trans.rigid_trans
        out.append((r.rot, r.t, r.scale, trans.v, sigma2, alpha, sdiag))
    return out


def _lowrank_loop(src, tgt, lmd, k, w, sigma2, iters, rank, power_iters=2, seed=0):
    """the device loop; returns (states as _oracle_loop, Q, Bc)"""
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_lowrank_begin(1.0, lmd, k, sigma2, w, rank, power_iters, seed)
    q, bc = h.bcpd_lowrank_factors()
    out = []
    for _ in range(iters):
        s2 = h.bcpd_step()
        rot, t, scale, sigma2_now, v, _, alpha, sdiag = h.bcpd_get(v=True, alpha=True, sigma_diag=True)
        assert s2 == sigma2_now
        out.append((rot, t, scale, v, sigma2_now, alpha, sdiag))
    return out, q, bc


def _compare(dev, ref, tol, rows=slice(None)):
    for it, (d, r) in enumerate(zip(dev, ref)):
        msg = "iteration %d" % it
        np.testing.assert_allclose(d[0], r[0], atol=tol, err_msg=msg)
        np.testing.assert_allclose(d[1], r[1], atol=tol * max(1.0, np.abs(r[1]).max()), err_msg=msg)
        assert d[2] == pytest.approx(r[2], rel=tol), msg
        np.testing.assert_allclose(d[3][rows], r[3][rows], atol=tol * max(1.0, np.abs(r[3]).max()), err_msg=msg)
        assert d[4] == pytest.approx(r[4], rel=tol), msg
        np.testing.assert_allclose(d[5][rows], r[5][rows], rtol=tol, err_msg=msg)
        np.testing.assert_allclose(d[6][rows], r[6][rows], rtol=tol, atol=tol * np.abs(r[6]).max(), err_msg=msg)


def _check_vs_oracle(m, case, rank, extent=2.0, iters=5, seed=3):
    """Both loops run the same E-step code on the same source order, and the oracle's M-step uses the device's own factors, so
    what may differ is the FP64 arithmetic of the M-step: the order of the sums over the points (St, Rt, v, diag Sigma, the moments)
    and the K x K inverse (cuSOLVER's LU against numpy's eigh and inv).  C = (c I + St)^-1 has eigenvalues in (0, 1 / c]; the
    inverse moves by about cond(c I + St) 1e-16 relative and the sums by 1e-16 of their absolute terms, which stays below 1e-10 here
    (cond <= 1e5 for these clouds and iterations); the rest is the float32 E-step seeing moved points that differ in their last
    FP64 bits.  TOL = 1e-6 (as in the dense loop's comparison) keeps a wide margin while a wrong ratio, a missing 1 / ratio on
    diag Sigma, or a transposed C Qt^T (all O(1) changes) cannot pass."""
    dim, w, k, lmd = case
    src, tgt = _box_pair(m, dim, extent, seed)
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    dev, q, bc = _lowrank_loop(src, tgt, lmd, k, w, sigma2, iters, rank)
    _compare(dev, _oracle_loop(src, tgt, q, bc, lmd, k, w, sigma2, iters), TOL)


# ---- 2. K = M against the dense loop -----------------------------------------------------------------------------------------------
def _check_full_rank(m, seed=3):
    """_pair's clouds spread to a spacing of about four units, where G^-1 is well conditioned: at K = M the low-rank loop solves the
    dense loop's system.  The two differ by their G: the dense loop inverts the float32 kernel matrix on the host, the low-rank one
    factors G from the float32 G X products (2^-23 relative per entry); cond(G) amplifies both into G^-1 and v.  The tolerance is
    cond(G) 2^-24 (at least 1e-6).  At M = 300 cond(G) is 434 (tolerance 2.6e-5) and the largest relative difference over four
    iterations 3.4e-7; at half the spacing cond(G) is 3750 and the difference 4.6e-6, at a quarter 6.7e4 and 2e-5 -- it follows
    cond(G) 2^-24 at 1/200 .. 1/75 of it."""
    dim, w, k, lmd = CASES[1]
    src, tgt = _pair(m, dim, seed)
    src, tgt = 4.0 * src, 4.0 * tgt
    cond = np.linalg.cond(_imq64(src, src))
    tol = max(1e-6, cond * U)
    print("K = M = %d: cond(G) = %.3g, tolerance %.3g" % (m, cond, tol))
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    dense = _device_loop(src, tgt, _gmat_inv(src), lmd, k, w, sigma2, 4)
    low, q, _ = _lowrank_loop(src, tgt, lmd, k, w, sigma2, 4, m)
    assert q.shape == (m, m)
    _compare(low, dense, tol)


# ---- 3. the IMQ G X product element by element -------------------------------------------------------------------------------------
def _imq_handle(src, c):
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(src[:64])
    h.bcpd_lowrank_begin(c, 2.0, 1e20, 0.1, 0.0, 1, 0, 1)
    return h


def _imq_tolerance(src, c, x, kernels):
    """Per-element bounds on |kernel(G X) - G64 X| over all rows; returns (G64 X, {kernel: bound}).

    Both kernels evaluate the same float32 tile value G' = min(1, rsqrt.approx(fl(1 + u))) in the frame a = fl(sb fl(y)),
    sb = fl(1 / sqrt(c)), u = |a_i - a_j|^2 by an FMA chain, and scale the FP64 result by gscale = 1 / sqrt(c).  Against
    G'64 = (1 + u64)^(-1/2):
      - coordinates and u as for the Gaussian kernel (test_zz_gram_product._tolerance): |du| <= 8 2^-24 u + 2^-21 A sqrt(D u)
        + D 2^-44 A^2 (A = sb max |y|), and |dG'/du| = G'^3 / 2, so a relative error of G'^2 |du| / 2 = |du| / (2 (1 + u));
      - fl(1 + u): 2^-24 relative on 1 + u, 2^-25 on G';  rsqrt.approx.ftz.f32: 2^-22.9 relative (1 / sqrtf in the emulation:
        two roundings, 2^-23);  the clamp to 1 only moves G' towards G'64 <= 1;
    so t1 = 1.01 G'64 (2^-22.9 + 2^-25 + |du| / (2 (1 + u))) (1.01: second-order terms).  From there the digit and float32-sum
    terms of the Gaussian bound apply unchanged to G' X, and every term is multiplied by gscale (its FP64 rounding and the FP64 join:
    2^-50 of sum G64 |X|)."""
    m, dim = src.shape
    sb = 1.0 / math.sqrt(c)
    a_max = sb * np.abs(src).max()
    ax = np.abs(x)
    colmax = ax.max(0)
    want = np.empty((m, x.shape[1]))
    tol = {k: np.empty_like(want) for k in kernels}
    for b0 in range(0, m, 256):
        r = np.arange(b0, min(m, b0 + 256))
        d2 = ((src[r][:, None, :] - src[None, :, :]) ** 2).sum(-1)
        u = d2 / c
        g64 = 1.0 / np.sqrt(1.0 + u)
        du = 8.0 * U * u + 2.0 ** -21 * a_max * np.sqrt(dim * u) + dim * 2.0 ** -44 * a_max ** 2
        t1 = 1.01 * g64 * (2.0 ** -22.9 + 2.0 ** -25 + du / (2.0 * (1.0 + u)))
        want[r] = sb * g64.dot(x)
        gx = g64.dot(ax)
        t1x = t1.dot(ax)
        if TC in kernels:
            xq = ax + 2.0 ** -23 * colmax
            gu = np.floor(2.0 ** 23 * (g64 + t1) + 0.5)
            a1, a2 = np.minimum(255.0, np.floor(gu / 256.0)), np.minimum(255.0, gu)
            lv34 = (2.0 ** 15 * (a1 + a2) + 2.0 ** 7 * a2).sum(1)
            tol[TC][r] = sb * (t1x + 2.0 ** -23 * colmax * t1.sum(1)[:, None] + U * xq.sum(0)[None, :]
                               + 2.0 ** -23 * colmax[None, :] * (g64 + t1 + U).sum(1)[:, None]
                               + 2.0 ** -45 * colmax[None, :] * lv34[:, None] + 2.0 ** -50 * gx)
        if CC in kernels:
            ex = (gx + t1x) * (1.0 + U)
            tol[CC][r] = sb * (t1x * (1.0 + U) + U * (gx + t1x) + (32.0 * U + 2.0 ** -53 * (m / 32.0 + 16.0)) * ex * (1.0 + 64.0 * U)
                               + 2.0 ** -50 * gx)
    return want, tol


def _smooth_columns(m, cols, seed):
    x = np.random.default_rng(seed).standard_normal((m, cols))
    x[:, 0] = 1.0
    return x


def _check_imq_product(m, kernels, cs=(1.0, 0.25, 4.0)):
    src, _ = _box_pair(m, 3, 3.0, 31)
    x = _smooth_columns(m, 70, 11)
    for c in cs:
        h = _imq_handle(src, c)
        want, tol = _imq_tolerance(src, c, x, kernels)
        got = {}
        for kern in kernels:
            got[kern] = h.lowrank_gram_product(x, kern)
            ratio = np.abs(got[kern] - want) / tol[kern]
            print("IMQ G X vs float64, kernel %d, M = %d, c = %g: worst |error| / tolerance = %.3g" % (kern, m, c, ratio.max()))
            assert ratio.max() <= 1.0, (kern, c)
        if len(kernels) == 2:
            assert np.all(np.abs(got[TC] - got[CC]) <= tol[TC] + tol[CC]), c
        # the row shares of a multi-rank handle add up exactly to the full product
        for kern in kernels:
            for world in (2, 3, 8):
                parts = [h.lowrank_gram_product(x, kern, world=world, rank=r) for r in range(world)]
                assert np.array_equal(np.sum(parts, axis=0), got[kern]), (kern, world, c)


def test_imq_bound_rejects_a_missing_scale():
    """A float32 restatement of the CUDA-core kernel (tile values, 32-term float32 sums, FP64 beyond) is within the bound with the
    1 / sqrt(c) scale and far outside it without (c = 4: a factor of 2)."""
    m, c = 600, 4.0
    src, _ = _box_pair(m, 3, 3.0, 31)
    x = _smooth_columns(m, 6, 3)
    want, tol = _imq_tolerance(src, c, x, (CC,))
    tol = tol[CC]
    a = np.float32(1.0 / math.sqrt(c)) * src.astype(np.float32)
    u = sum((a[:, k][:, None] - a[None, :, k]) ** 2 for k in range(3)).astype(np.float32)
    e = np.minimum(np.float32(1.0), np.float32(1.0) / np.sqrt(np.float32(1.0) + u))
    xf = x.astype(np.float32)
    raw = sum(e[:, j0:j0 + 32].dot(xf[j0:j0 + 32]).astype(np.float64) for j0 in range(0, m, 32))
    assert (np.abs(raw / math.sqrt(c) - want) / tol).max() <= 1.0
    assert (np.abs(raw - want) / tol).max() > 1e3


# ---- 4. factor quality -----------------------------------------------------------------------------------------------------------------
def _factor_error(src, rank):
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(src[:64])
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, rank, 2, 0)
    q, bc = h.bcpd_lowrank_factors()
    g = _imq64(src, src)
    return np.linalg.norm(g - q.dot(bc).dot(q.T), 2) / np.linalg.norm(g, 2)


def _check_factor_quality(m, rank_unit, ranks_box3):
    rng = np.random.default_rng(41)
    err = _factor_error(rng.random((m, 3)), rank_unit)
    print("extent 1, M = %d, K = %d: |G - Q Bc Q^T| / |G| = %.3g" % (m, rank_unit, err))
    assert err <= 1e-6
    box3 = 3.0 * rng.random((m, 3))
    errs = [_factor_error(box3, k) for k in ranks_box3]
    print("extent 3, M = %d, K = %s: %s" % (m, ranks_box3, ["%.3g" % e for e in errs]))
    assert all(b < a for a, b in zip(errs, errs[1:])), errs


# ---- 5. where the dense loop fails ------------------------------------------------------------------------------------------------------
def _check_dense_fails(m):
    """A source of extent 0.5 (c = 1; the bunny of the reference's example spans about 0.2): G is numerically of rank about 10-40
    and its float32 inverse is rounding noise -- far from symmetric positive definite, its symmetric part has negative eigenvalues
    as large as its positive ones.  The dense loop shows it (a refused step, a negative diag Sigma or a sigma2 that is not
    positive; here a negative diag Sigma in the first step), the low-rank loop runs 30 iterations with diag Sigma >= 0 and a
    positive finite sigma2.  lmd = 20: with lmd = 2 the prior lets v (whose kernel is nearly flat over so small a cloud) take over
    the similarity; the scale of the low-rank loop then drifts towards 0 until a step is refused.  A source no target explains (nu = 0) keeps a finite v."""
    src, tgt = _box_pair(m, 3, 0.5, 43)
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    ginv = np.ascontiguousarray(np.linalg.inv(math_utils.inverse_multiquadric_kernel(src, src)))
    eig = np.linalg.eigvalsh(0.5 * (ginv + ginv.T).astype(np.float64))
    assert eig[0] < -1e-3 * eig[-1]
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_begin(ginv, 20.0, 1e20, sigma2, 0.05)
    failed = None
    for it in range(30):
        try:
            s2 = h.bcpd_step()
        except _cabi.CpdError as e:
            failed = "step %d refused: %s" % (it, e)
            break
        sd = h.bcpd_get(v=False, sigma_diag=True)[7]
        if sd.min() < 0.0 or not (0.0 < s2 < np.inf):
            failed = "step %d: min diag Sigma %.3g, sigma2 %.3g" % (it, sd.min(), s2)
            break
    print("dense loop on a cloud of extent 0.5:", failed)
    assert failed is not None
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_lowrank_begin(1.0, 20.0, 1e20, sigma2, 0.05, 100, 2, 0)
    for _ in range(30):
        s2 = h.bcpd_step()
        assert 0.0 < s2 < np.inf
        rot, t, scale, _, v, _, alpha, sd = h.bcpd_get(v=True, alpha=True, sigma_diag=True)
        assert sd.min() >= 0.0 and np.all(np.isfinite(v)) and np.all(np.isfinite(alpha)) and np.isfinite(scale)
    # a source far from every target: nu = 0 exactly, its v stays finite
    src, tgt = _box_pair(m, 3, 0.5, 43, far=True)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_lowrank_begin(1.0, 20.0, 1e20, sigma2, 0.05, 100, 2, 0)
    for _ in range(3):
        assert 0.0 < h.bcpd_step() < np.inf
        v, sd = h.bcpd_get(v=True, sigma_diag=True)[4::3]
        assert h.last_estep()[1][-1] == 0.0
        assert np.all(np.isfinite(v)) and sd.min() >= 0.0


# ---- 6. refusals and the shared factors -----------------------------------------------------------------------------------------------
def _check_state():
    src, tgt = _box_pair(200, 3, 2.0, 47)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    for args in ((1.0, 0), (1.0, 1025), (0.0, 10), (-1.0, 10), (float("inf"), 10)):
        with pytest.raises(ValueError):
            h.bcpd_lowrank_begin(args[0], 2.0, 1e20, 0.1, 0.0, args[1])
    for pi in (-1, 9):
        with pytest.raises(ValueError):
            h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 10, pi)
    lib = _cabi.lib() if _cabi._lib is None else _cabi._lib
    for c, rank, pi in ((0.0, 10, 2), (1.0, 0, 2), (1.0, 1025, 2), (1.0, 10, 9), (1.0, 10, -1)):
        assert lib.cpd_bcpd_lowrank_begin(h._h, c, 2.0, 1e20, 0.1, 0.0, rank, pi, 0) == -1          # CPD_ERR_ARG
    with pytest.raises(_cabi.CpdError, match="lowrank_begin has not been called"):
        h.bcpd_lowrank_factors()
    # rank clamped to M
    small = _cabi.Handle(3)
    small.set_source(src[:20])
    small.set_target(tgt)
    small.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 50)
    assert small.bcpd_lowrank_factors()[0].shape == (20, 20)
    small.bcpd_step()
    # a step after the source changed
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    h.bcpd_step()
    h.set_source(src[:-1])
    with pytest.raises(_cabi.CpdError, match="size changed"):
        h.bcpd_step()
    # the same source set again: a new begin is needed
    h.set_source(src)
    with pytest.raises(_cabi.CpdError, match="begin"):
        h.bcpd_step()
    x = _smooth_columns(200, 3, 5)
    # a non-rigid begin between two low-rank BCPD steps ends the BCPD loop, and the products apply the Gaussian from then on
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    h.bcpd_step()
    imq = h.lowrank_gram_product(x, CC)
    h.nonrigid_lowrank_begin(2.0, 2.0, 0.1, 0.0, 20)
    with pytest.raises(_cabi.CpdError, match="cpd_nonrigid_.*begin replaced the low-rank factors"):
        h.bcpd_step()
    with pytest.raises(_cabi.CpdError, match="replaced the low-rank factors"):
        h.bcpd_lowrank_factors()
    gauss = h.lowrank_gram_product(x, CC)
    d2 = ((src[:, None] - src[None]) ** 2).sum(-1)
    np.testing.assert_allclose(gauss, np.exp(-d2 / 4.0).dot(x), rtol=0, atol=1e-5 * np.abs(x).sum(0).max())
    np.testing.assert_allclose(imq, _imq64(src, src).dot(x), rtol=0, atol=1e-5 * np.abs(x).sum(0).max())
    h.nonrigid_step()
    # ... and the reverse: a low-rank BCPD begin ends the non-rigid loop
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    with pytest.raises(_cabi.CpdError, match="cpd_bcpd_lowrank_begin replaced the low-rank factors"):
        h.nonrigid_step()
    np.testing.assert_array_equal(h.lowrank_gram_product(x, CC), imq)
    h.bcpd_step()
    # a dense non-rigid begin ends the low-rank BCPD loop too
    h.nonrigid_begin(2.0, 2.0, 0.1, 0.0)
    with pytest.raises(_cabi.CpdError, match="replaced the low-rank factors"):
        h.bcpd_step()
    # a dense BCPD begin returns the handle to the dense loop: its steps equal a fresh handle's
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    h.bcpd_step()
    ginv = _gmat_inv(src)
    h.bcpd_begin(ginv, 2.0, 1e20, 0.1, 0.05)
    fresh = _cabi.Handle(3)
    fresh.set_source(src)
    fresh.set_target(tgt)
    fresh.bcpd_begin(ginv, 2.0, 1e20, 0.1, 0.05)
    for _ in range(2):
        assert h.bcpd_step() == fresh.bcpd_step()
    np.testing.assert_array_equal(h.bcpd_get()[4], fresh.bcpd_get()[4])


def _check_comm_refused():
    src, tgt = _box_pair(100, 3, 2.0, 19)
    comm = _cabi.comm_create(0, 1, 0, _cabi.unique_id())
    try:
        h = _cabi.Handle(3)
        h.set_source(src)
        h.set_target(tgt)
        h.attach_comm(comm, 1, 0)
        with pytest.raises(_cabi.CpdError, match="communicator"):
            h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 10)
        h.close()
    finally:
        _cabi.comm_destroy(comm)


# ---- 8. Python surface -------------------------------------------------------------------------------------------------------------
class _HostMstep(bcpd.CombinedBCPD):
    def maximization_step(self, target, rigid_trans, estep_res, sigma2_p=None):
        return super(_HostMstep, self).maximization_step(target, rigid_trans, estep_res, sigma2_p)


class _HostEstep(bcpd.CombinedBCPD):
    def expectation_step(self, *args, **kwargs):
        return super(_HostEstep, self).expectation_step(*args, **kwargs)


def _check_python(m, rank):
    src, tgt = _box_pair(m, 3, 2.0, 53)
    for cls in (_HostMstep, _HostEstep):
        with pytest.raises(ValueError, match="low_rank"):
            cls(src, low_rank=rank)
    for bad in (0, -3, 2.5, True):
        with pytest.raises(ValueError):
            bcpd.CombinedBCPD(src, low_rank=bad)
    reg = bcpd.CombinedBCPD(src, low_rank=rank)
    with pytest.raises(ValueError, match="dense only"):
        reg.maximization_step(tgt, None, None)
    # registration_bcpd(low_rank=K) against the Handle-driven loop with the reference's stopping criterion
    w, maxiter, tol = 0.05, 40, 2e-3
    seen = []
    out = bcpd.registration_bcpd(src, tgt, w=w, maxiter=maxiter, tol=tol, low_rank=rank, low_rank_iters=1, low_rank_seed=7,
                                 callbacks=[lambda t: seen.append(np.array(t.v, copy=True))])
    assert reg.gmat is None if hasattr(reg, "gmat") else True
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, math_utils.squared_kernel_sum(src, tgt), w, rank, 1, 7)
    from scipy.spatial import cKDTree
    tree = cKDTree(tgt, leafsize=10)
    previous, vs = None, []
    for _ in range(maxiter):
        moved = h.bcpd_get(v=False, moved=True)[5]
        h.bcpd_step()
        vs.append(h.bcpd_get()[4])
        crit = math_utils.compute_rmse(moved, tree)
        if previous is not None and abs(previous - crit) < tol:
            break
        previous = crit
    assert 1 < len(seen) < maxiter and len(seen) == len(vs)
    for a, b in zip(seen, vs):
        np.testing.assert_array_equal(a, b)
    rot, t, scale = h.bcpd_get()[:3]
    np.testing.assert_array_equal(out.rigid_trans.rot, rot)
    np.testing.assert_array_equal(out.rigid_trans.t, t)
    assert out.rigid_trans.scale == scale
    np.testing.assert_array_equal(out.v, vs[-1])
    solver = bcpd.CombinedBCPD(src, low_rank=rank)
    solver.registration(tgt, maxiter=1)
    assert solver.gmat is None and solver.gmat_inv is None


# ---- CPU: the CPU emulation of the library -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_bcpd_lowrank_vs_oracle_emulated(emulated, case):
    _check_vs_oracle(400 if case[0] == 3 else 300, case, 60)


def test_bcpd_lowrank_full_rank_equals_dense_emulated(emulated):
    _check_full_rank(300)


def test_imq_gram_product_emulated(emulated):
    _check_imq_product(500, (CC,))


def test_bcpd_lowrank_factor_quality_emulated(emulated):
    _check_factor_quality(500, 100, (20, 40, 80))


def test_bcpd_lowrank_where_dense_fails_emulated(emulated):
    _check_dense_fails(300)


def test_bcpd_lowrank_state_emulated(emulated):
    _check_state()


def test_bcpd_lowrank_refuses_a_communicator_emulated(emulated):
    _check_comm_refused()


def test_bcpd_lowrank_python_emulated(emulated):
    _check_python(300, 40)


def test_imq_tensor_core_product_is_refused_emulated(emulated):
    src, _ = _box_pair(100, 3, 2.0, 59)
    h = _imq_handle(src, 1.0)
    with pytest.raises(_cabi.CpdError, match="no tensor-core"):
        h.lowrank_gram_product(np.ones((100, 2)), TC)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("m", [4000, 20000])
@pytest.mark.parametrize("case", CASES)
def test_bcpd_lowrank_vs_oracle_gpu(case, m):
    _check_vs_oracle(m, case, 200 if m > 4000 else 120)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_lowrank_full_rank_equals_dense_gpu():
    _check_full_rank(1000)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_imq_gram_product_gpu():
    """17000 points: two j-chunks of the tensor-core kernel, both kernels, three values of c."""
    _check_imq_product(17000, (TC, CC))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_lowrank_factor_quality_gpu():
    _check_factor_quality(2000, 100, (50, 100, 200))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_lowrank_where_dense_fails_gpu():
    _check_dense_fails(2000)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_lowrank_state_gpu():
    _check_state()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_lowrank_python_gpu():
    _check_python(3000, 100)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_bcpd_lowrank_100k_gpu():
    """100 000 points at K = 200 through registration_bcpd(low_rank=200, maxiter=20): sigma2 positive and finite, the handle's
    device memory (cudaMemGetInfo before and after) under 2 GB -- the dense loop would need about 20 M^2 = 200 GB -- and two runs
    with the same seed give bit-identical v."""
    torch = pytest.importorskip("torch")
    m = 100000
    src, tgt = _box_pair(m, 3, 2.0, 61)
    free0 = torch.cuda.mem_get_info(0)[0]
    reg = bcpd.CombinedBCPD(src, low_rank=200)
    out = reg.registration(tgt, w=0.05, maxiter=20, tol=-1.0)
    free1 = torch.cuda.mem_get_info(0)[0]
    used = free0 - free1
    sigma2 = reg._h.bcpd_get(v=False)[3]
    print("100k, K = 200: handle device memory %.3f GB, sigma2 %.4g" % (used / 2.0 ** 30, sigma2))
    assert 0.0 < sigma2 < np.inf
    assert used < 2 * 2 ** 30
    assert np.all(np.isfinite(out.v))
    again = bcpd.registration_bcpd(src, tgt, w=0.05, maxiter=20, tol=-1.0, low_rank=200)
    np.testing.assert_array_equal(out.v, again.v)
