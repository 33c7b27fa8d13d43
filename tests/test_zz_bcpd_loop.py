"""The BCPD registration loop on the device (cpd_bcpd_begin / step / get, CombinedBCPD.registration) against the host loop.

The host loop is the library's weighted E-step (cpd_bcpd_estep on a handle whose source is the ORIGINAL source, so that both loops
sum the pair terms in the same internal order) followed by ``CombinedBCPD._maximization_step`` -- the numpy M-step pinned to the
reference by test_zz_bcpd.py.  Both are fed the same float32 G^-1.  What may differ is the order of the FP64 arithmetic of the M-step
(cuSOLVER's pivoting and the internal point order against LAPACK's inverse) and the last bit of a moved point before its rounding to
float32 in the E-step; replaying the host M-step with a randomly permuted LU moves rot, t, scale and v by at most 4e-9 and sigma2 by
1.5e-9 relative over 5-8 iterations, so TOL = 1e-6 leaves a margin of about 250 while a transposed or one-sidedly permuted G^-1 (O(1)
changes) cannot pass.  CPU tests run the bodies under the emulation of tests/emu (M <= 500); the gpu-marked ones on the H100.
"""
import numpy as np
import pytest
from scipy.special import digamma

from oracle import cpd_oracle as orc
from probreg_b200 import _cabi, bcpd, math_utils
from probreg_b200 import transformation as tf

TOL = 1e-6


def _pair(m, dim, seed, far=False):
    """A source in random order and a rotated, scaled, smoothly deformed and noised target with a different count.  far: the
    last source sits far from every target (nu = 0 exactly).  The points are about one unit apart: on a denser cloud the float32
    inverse of the IMQ kernel matrix (c = 1) is so far from symmetric positive definite that diag(Sigma) turns negative for some
    sources, which the E-step of the host loop refuses.  On these clouds diag(Sigma) stays positive in every case that runs."""
    rng = np.random.default_rng(seed)
    side = m ** (1.0 / dim) / (0.7 * 0.4) ** (1.0 / 3.0) if dim == 3 else m ** 0.5 / 0.7 ** 0.5
    src = rng.random((m, dim)) * (side * np.array([1.0, 0.7, 0.4][:dim]))
    rot = orc.rot_z(20.0)[:dim, :dim]
    n = m + 37
    base = np.concatenate([src, rng.random((n - m, dim)) * 0.8 * side])[rng.permutation(n)]
    tgt = 1.05 * base.dot(rot.T) + side * np.array([0.1, -0.2, 0.15][:dim])
    tgt = tgt + 0.02 * side * np.sin(3.0 * tgt[:, ::-1] / side) + 0.01 * rng.standard_normal((n, dim))
    if far:
        src[-1] = 100.0 * side
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)


def _gmat_inv(src):
    return np.linalg.inv(orc.imq_kernel_f32(src, src, 1.0))


def _targets(tgt, iters):
    """tgt: one target for every iteration, or a list of one per iteration"""
    return tgt if isinstance(tgt, list) else [tgt] * iters


def _host_loop(src, tgt, ginv, lmd, k, w, sigma2, iters):
    """[(rot, t, scale, v, sigma2, alpha, sigma_diag)] per iteration: library E-step + the host M-step.  A source with nu = 0 gets
    x_hat = 0 (its residual is multiplied by nu = 0; the reference would carry the nan of 0 / 0 into every v)."""
    dim = src.shape[1]
    h = _cabi.Handle(dim)
    h.set_source(src)
    trans = tf.CombinedTransformation(np.identity(dim), np.zeros(dim))
    alpha, sdiag = np.full(src.shape[0], 1.0 / src.shape[0]), np.ones(src.shape[0])
    out, last = [], None
    for tgt in _targets(tgt, iters):
        if tgt is not last:
            h.set_target(tgt)
            last = tgt
        moved = trans.transform(src)
        nu_d, nu, px, n_p = h.bcpd_estep(moved, trans.rigid_trans.scale, alpha, sdiag, sigma2, w)
        with np.errstate(divide="ignore", invalid="ignore"):
            x_hat = np.where(nu[:, None] > 0, px / nu[:, None], 0.0)
        es = bcpd.EstepResult(nu_d, nu, n_p, px, x_hat)
        res = bcpd.CombinedBCPD._maximization_step(src, tgt, trans.rigid_trans, es, ginv, lmd, k, sigma2)
        trans, alpha, sdiag, sigma2 = res.transformation, res.alpha, res.sigma_mat.diagonal().copy(), res.sigma2
        r = trans.rigid_trans
        out.append((r.rot, r.t, r.scale, trans.v, sigma2, alpha, sdiag))
    return out


def _device_loop(src, tgt, ginv, lmd, k, w, sigma2, iters):
    tgts = _targets(tgt, iters)
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(tgts[0])
    h.bcpd_begin(ginv, lmd, k, sigma2, w)
    out, last = [], tgts[0]
    for tgt in tgts:
        if tgt is not last:
            h.set_target(tgt)            # a new target between two steps: the loop carries on from its state
            last = tgt
        s2 = h.bcpd_step()
        rot, t, scale, sigma2, v, _, alpha, sdiag = h.bcpd_get(v=True, alpha=True, sigma_diag=True)
        assert s2 == sigma2
        out.append((rot, t, scale, v, sigma2, alpha, sdiag))
    return out


def _compare(dev, host, tol=TOL, rows=slice(None)):
    for it, (d, r) in enumerate(zip(dev, host)):
        msg = "iteration %d" % it
        np.testing.assert_allclose(d[0], r[0], atol=tol, err_msg=msg)
        np.testing.assert_allclose(d[1], r[1], atol=tol, err_msg=msg)
        assert d[2] == pytest.approx(r[2], rel=tol), msg
        np.testing.assert_allclose(d[3][rows], r[3][rows], atol=tol, err_msg=msg)
        assert d[4] == pytest.approx(r[4], rel=tol), msg
        np.testing.assert_allclose(d[5][rows], r[5][rows], rtol=tol, err_msg=msg)
        np.testing.assert_allclose(d[6][rows], r[6][rows], rtol=tol, err_msg=msg)


# (dim, w, k, lmd): every value of each parameter, in both dimensions
CASES = [(3, 0.0, 1e20, 2.0), (3, 0.05, 1.0, 0.5), (3, 0.2, 1e20, 0.5), (2, 0.0, 1.0, 2.0), (2, 0.05, 1e20, 2.0), (2, 0.2, 1.0, 0.5)]


def _check_vs_host(m, case, iters=5, seed=3):
    dim, w, k, lmd = case
    src, tgt = _pair(m, dim, seed)
    ginv = _gmat_inv(src)
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    _compare(_device_loop(src, tgt, ginv, lmd, k, w, sigma2, iters), _host_loop(src, tgt, ginv, lmd, k, w, sigma2, iters))


def _check_orientation(m):
    """A deliberately non-symmetric G^-1 (the symmetric part of the true inverse plus an antisymmetric 1 % perturbation), fed to both
    loops, must agree; the same matrix transposed on the device side only must not."""
    dim, w, k, lmd = 3, 0.05, 1e20, 2.0
    src, tgt = _pair(m, dim, 5)
    g = _gmat_inv(src).astype(np.float64)
    g = 0.5 * (g + g.T)
    rng = np.random.default_rng(9)
    e = rng.standard_normal(g.shape)
    e = e - e.T
    g = g + 0.01 * np.abs(g).max() / np.abs(e).max() * e
    ginv = np.ascontiguousarray(g.astype(np.float32))
    assert np.abs(ginv - ginv.T).max() > 1e-3 * np.abs(ginv).max()
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    host = _host_loop(src, tgt, ginv, lmd, k, w, sigma2, 3)
    _compare(_device_loop(src, tgt, ginv, lmd, k, w, sigma2, 3), host)
    with pytest.raises(AssertionError):
        _compare(_device_loop(src, tgt, np.ascontiguousarray(ginv.T), lmd, k, w, sigma2, 3), host)


def _check_alpha():
    src, tgt = _pair(300, 3, 7)
    ginv = _gmat_inv(src)
    for k in (1e20, 1.0, 0.01):
        h = _cabi.Handle(3)
        h.set_source(src)
        h.set_target(tgt)
        h.bcpd_begin(ginv, 2.0, k, 0.1, 0.05)
        h.bcpd_step()
        alpha = h.bcpd_get(v=False, alpha=True)[6]
        _, nu, _, n_p = h.last_estep()
        ref = np.exp(digamma(k + nu) - digamma(k * src.shape[0] + n_p))
        np.testing.assert_allclose(alpha, ref, rtol=1e-12, atol=0)


class _HostLoopBCPD(bcpd.CombinedBCPD):
    """Overrides maximization_step, so registration() keeps the host loop (as a user's own M-step would)."""

    def maximization_step(self, target, rigid_trans, estep_res, sigma2_p=None):
        return super(_HostLoopBCPD, self).maximization_step(target, rigid_trans, estep_res, sigma2_p)


def _check_callbacks_and_stopping():
    src, tgt = _pair(300, 3, 11)
    runs = []
    for cls in (bcpd.CombinedBCPD, _HostLoopBCPD):
        seen = []
        reg = cls(src, lmd=2.0)
        assert reg._has_device_loop() == (cls is bcpd.CombinedBCPD)
        reg.set_callbacks([lambda t: seen.append((t.rigid_trans.rot.copy(), t.rigid_trans.t.copy(), t.rigid_trans.scale,
                                                  np.array(t.v, copy=True)))])
        out = reg.registration(tgt, w=0.05, maxiter=40, tol=2e-3)
        runs.append((seen, out))
    (dev_seen, dev), (host_seen, host) = runs
    assert 1 < len(dev_seen) < 40 and len(dev_seen) == len(host_seen)
    # the host loop's E-step sums the pair terms in the order of the MOVED source, so the two differ by the float32 rounding of
    # the E-step (1e-7 relative per sum): the tolerance of the registration test in test_zz_bcpd.py
    for d, r in zip(dev_seen, host_seen):
        np.testing.assert_allclose(d[0], r[0], atol=1e-5)
        np.testing.assert_allclose(d[1], r[1], atol=1e-5)
        assert d[2] == pytest.approx(r[2], rel=1e-5)
        np.testing.assert_allclose(d[3], r[3], atol=1e-5)
    assert isinstance(dev, tf.CombinedTransformation)
    np.testing.assert_allclose(dev.transform(src), host.transform(src), atol=1e-5)
    np.testing.assert_array_equal(dev.v, dev_seen[-1][3])


def _check_edges():
    # a source far from every target: nu = 0 exactly, v stays finite there and the other sources follow the host loop
    src, tgt = _pair(300, 3, 13, far=True)
    ginv = _gmat_inv(src)
    dev = _device_loop(src, tgt, ginv, 2.0, 1e20, 0.05, 1.0, 3)
    host = _host_loop(src, tgt, ginv, 2.0, 1e20, 0.05, 1.0, 3)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.bcpd_begin(ginv, 2.0, 1e20, 1.0, 0.05)
    h.bcpd_step()
    assert h.last_estep()[1][-1] == 0.0
    for d in dev:
        assert all(np.all(np.isfinite(a)) for a in (d[0], d[1], d[3], d[5], d[6]))
    _compare(dev, host)
    # sigma2 that is not a positive finite number: every target column dead in the first E-step (n_p = 0)
    src, tgt = _pair(200, 3, 17)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt + 100.0)
    h.bcpd_begin(_gmat_inv(src), 2.0, 1e20, 1e-6, 0.05)
    with pytest.raises(_cabi.CpdError, match="sigma2 = "):
        h.bcpd_step()
    with pytest.raises(_cabi.CpdError, match="stopped on an error.*begin again"):
        h.bcpd_step()
    # an exactly singular precision matrix: G^-1 = 0 and a source with nu = 0 leave a zero column; getrf's info is reported
    src_far, tgt_far = _pair(200, 3, 13, far=True)
    h = _cabi.Handle(3)
    h.set_source(src_far)
    h.set_target(tgt_far)
    h.bcpd_begin(np.zeros((200, 200), dtype=np.float32), 2.0, 1e20, 1.0, 0.05)
    with pytest.raises(_cabi.CpdError, match="getrf info = [1-9]"):
        h.bcpd_step()
    with pytest.raises(_cabi.CpdError, match="stopped on an error"):
        h.bcpd_step()
    h.bcpd_begin(_gmat_inv(src_far), 2.0, 1e20, 1.0, 0.05)          # a new begin starts over
    assert h.bcpd_step() > 0.0
    # step before begin, a wrong gmat_inv, a changed source, a communicator
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    with pytest.raises(_cabi.CpdError, match="begin"):
        h.bcpd_step()
    ginv = _gmat_inv(src)
    for bad in (ginv[:-1], ginv[:, :-1], ginv.astype(np.float64), np.asfortranarray(ginv), ginv.tolist()):
        with pytest.raises(ValueError):
            h.bcpd_begin(bad, 2.0, 1e20, 0.1, 0.0)
    h.bcpd_begin(ginv, 2.0, 1e20, 0.1, 0.0)
    h.bcpd_step()
    h.set_source(src[:-1])
    with pytest.raises(_cabi.CpdError, match="size changed"):
        h.bcpd_step()


def _check_target_reset():
    """The target may be set again between two steps, with any count (here 300 -> 3000 points); the loop goes on from its state
    exactly like the host loop given the same targets."""
    src, tgt = _pair(300, 3, 23)
    rng = np.random.default_rng(29)
    tgt_big = np.ascontiguousarray(tgt[rng.integers(0, tgt.shape[0], 3000)] + 0.05 * rng.standard_normal((3000, 3)))
    tgts = [tgt, tgt_big, tgt_big, tgt]
    ginv = _gmat_inv(src)
    sigma2 = math_utils.squared_kernel_sum(src, tgt)
    _compare(_device_loop(src, tgts, ginv, 2.0, 1e20, 0.05, sigma2, 4), _host_loop(src, tgts, ginv, 2.0, 1e20, 0.05, sigma2, 4))


def _check_comm_refused():
    src, tgt = _pair(100, 3, 19)
    uid = _cabi.unique_id()
    comm = _cabi.comm_create(0, 1, 0, uid)
    try:
        h = _cabi.Handle(3)
        h.set_source(src)
        h.set_target(tgt)
        h.attach_comm(comm, 1, 0)
        with pytest.raises(_cabi.CpdError, match="communicator"):
            h.bcpd_begin(_gmat_inv(src), 2.0, 1e20, 0.1, 0.0)
        with pytest.raises(_cabi.CpdError, match="communicator"):
            h.bcpd_step()
        h.close()
    finally:
        _cabi.comm_destroy(comm)


# ---- CPU: the CPU emulation of the library -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_bcpd_loop_vs_host_emulated(emulated, case):
    _check_vs_host(400 if case[0] == 3 else 300, case)


def test_bcpd_loop_orientation_emulated(emulated):
    _check_orientation(300)


def test_bcpd_loop_alpha_emulated(emulated):
    _check_alpha()


def test_bcpd_loop_callbacks_and_stopping_emulated(emulated):
    _check_callbacks_and_stopping()


def test_bcpd_loop_edges_emulated(emulated):
    _check_edges()


def test_bcpd_loop_target_reset_emulated(emulated):
    _check_target_reset()


def test_bcpd_loop_refuses_a_communicator_emulated(emulated):
    _check_comm_refused()


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("m", [1500, 4000])
@pytest.mark.parametrize("case", CASES)
def test_bcpd_loop_vs_host_gpu(case, m):
    _check_vs_host(m, case)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_loop_orientation_gpu():
    _check_orientation(1500)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_loop_alpha_gpu():
    _check_alpha()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_loop_callbacks_and_stopping_gpu():
    _check_callbacks_and_stopping()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_loop_edges_gpu():
    _check_edges()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_bcpd_loop_target_reset_gpu():
    _check_target_reset()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_bcpd_loop_10k_gpu():
    """M = N = 10k (the target here has M + 37 points), three iterations against the host loop: tens of seconds of host LAPACK."""
    _check_vs_host(10000, CASES[0], iters=3)
