"""Low-rank non-rigid CPD (BASELINE configuration 5) and the device-side correspondence priors.

There is no reference counterpart for the low-rank path (the reference solves the dense M x M system, cpd.py:296), so
parity is anchored against the reference's dense arithmetic (the numpy oracle) at sizes where the
dense solve is possible, with the truncation error of the factorisation as the tolerance, and -- tighter -- against the
oracle run on the SAME approximate G = Q Bc Q^T, where only rounding separates the two.

CPU tests run the library under the emulation of tests/emu; the gpu-marked ones call the real library.
"""
import os

import numpy as np
import pytest

from oracle import cpd_oracle as orc
from probreg_b200 import _cabi, cpd

F = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])


def _deformed_pair(m, seed=9):
    src, _ = orc.synthetic_pair(m)
    tgt = src + 0.03 * np.sin(2 * np.pi * src.dot(F)) + 0.002 * np.random.default_rng(seed).standard_normal(src.shape)
    return src, tgt


# ---- the algebra (numpy only) -----------------------------------------------------------------------------------------------
def test_kxk_form_equals_the_dense_solve_on_the_same_low_rank_g():
    src, tgt = _deformed_pair(300)
    q, bc = orc.lowrank_factors(src, 2.0, 40)
    g_lr = q.dot(bc).dot(q.T)
    es = orc.expectation_step(src, tgt, 0.01, 0.05)
    dense = orc.mstep_nonrigid(src, tgt, es, 0.01, g_lr, 1.5)
    lr = orc.mstep_nonrigid_lowrank(src, tgt, es, 0.01, q, bc, 1.5)
    np.testing.assert_allclose(lr.params[1], src + g_lr.dot(dense.params[0]), atol=1e-9)
    assert lr.sigma2 == pytest.approx(dense.sigma2, rel=1e-9)
    # W itself: T = Y + G W must hold for the low-rank W as well
    np.testing.assert_allclose(src + g_lr.dot(lr.params[0]), lr.params[1], atol=1e-9)
    # and with correspondence priors
    p1t, pxt = orc.constraint_terms(300, tgt, np.arange(0, 300, 15), np.arange(0, 300, 15))
    dense = orc.mstep_nonrigid(src, tgt, es, 0.01, g_lr, 1.5, alpha=1e-2, p1_tilde=p1t, px_tilde=pxt)
    lr = orc.mstep_nonrigid_lowrank(src, tgt, es, 0.01, q, bc, 1.5, alpha=1e-2, p1_tilde=p1t, px_tilde=pxt)
    np.testing.assert_allclose(lr.params[1], src + g_lr.dot(dense.params[0]), atol=1e-9)


def test_range_finder_reaches_float32_noise_quickly():
    src, _ = _deformed_pair(500)
    g = orc.rbf_kernel_f32(src, src, 2.0).astype(np.float64)
    for rank, bound in [(10, 1e-4), (40, 1e-7)]:
        q, bc = orc.lowrank_factors(src, 2.0, rank)
        assert np.linalg.norm(g - q.dot(bc).dot(q.T), 2) / np.linalg.norm(g, 2) < bound


# ---- the library (bodies shared by the emulated CPU tests and the GPU tests) ---------------------------------------------------
def _check_against_oracles(m, rank, iters, beta, lmd, w, tol_dense, constrained=False):
    src, tgt = _deformed_pair(m)
    kw = {}
    okw = {}
    if constrained:
        idx = np.arange(0, m, 11)
        kw = {"alpha": 1e-2, "idx_source": idx, "idx_target": idx}
        okw = {"alpha": 1e-2, "idx_source": idx, "idx_target": idx}
    cls = cpd.ConstrainedNonRigidCPD if constrained else cpd.NonRigidCPD
    reg = cls(src, beta=beta, lmd=lmd, low_rank=rank, **kw)
    res = reg.registration(tgt, w=w, maxiter=iters, tol=-1.0)
    moved = reg.moved_source()
    tfm = res.transformation
    k = min(rank, m)
    assert tfm.q.shape == (m, k) and tfm.bcore.shape == (k, k) and tfm.w.shape == (m, 3)
    # the factors: orthonormal columns (or zero ones once the numerical rank is exhausted), symmetric core
    gram = tfm.q.T.dot(tfm.q)
    d = np.diag(gram)
    assert np.all((np.abs(d - 1.0) < 1e-12) | (d == 0.0))
    np.testing.assert_allclose(gram - np.diag(d), 0.0, atol=1e-12)
    np.testing.assert_allclose(tfm.bcore, tfm.bcore.T, atol=0.0)
    g_lr = tfm.q.dot(tfm.bcore).dot(tfm.q.T)
    g = orc.rbf_kernel_f32(src, src, beta).astype(np.float64)
    assert np.linalg.norm(g - g_lr, 2) / np.linalg.norm(g, 2) < (1e-6 if k >= 30 else 1e-3)
    # the transformation object reproduces the device's moved points
    np.testing.assert_allclose(tfm.transform(src), moved, atol=1e-10)
    # 1. the reference's dense arithmetic on the SAME G: only rounding (and the FP32 pair maths of the E-step) differ
    tf_name = "nonrigid_constrained" if constrained else "nonrigid"
    same, _ = orc.registration(src, tgt, tf_name, maxiter=iters, tol=-1.0, beta=beta, lmd=lmd, w=w, g=g_lr, **okw)
    # (moved points at 1e-4: the FP32 pair arithmetic of the E-step perturbs P by ~1e-7 extent / sigma, and the solve of
    #  cpd.py:296 amplifies that -- more so for a wide kernel and thousands of points; measured under the emulation with a
    #  MUFU-like ex2: 2.8e-5 at M = 2000, beta = 2.  sigma2 stays tight.)
    assert res.sigma2 == pytest.approx(same.sigma2, rel=1e-5)
    np.testing.assert_allclose(moved, src + g_lr.dot(same.params[0]), atol=1e-4)
    # 2. the reference itself (exact G): the truncation error of the factorisation on top
    ref, _ = orc.registration(src, tgt, tf_name, maxiter=iters, tol=-1.0, beta=beta, lmd=lmd, w=w, **okw)
    assert res.sigma2 == pytest.approx(ref.sigma2, rel=tol_dense)
    np.testing.assert_allclose(moved, src + g.dot(ref.params[0]), atol=max(1e-4, tol_dense))
    return res


def _check_full_rank_equals_dense(m):
    """rank == M: the factorisation is exact up to rounding, so the low-rank loop must land on the dense device loop."""
    src, tgt = _deformed_pair(m)
    a = cpd.NonRigidCPD(src, beta=0.5, lmd=1.0)
    ra = a.registration(tgt, w=0.0, maxiter=4, tol=-1.0)
    b = cpd.NonRigidCPD(src, beta=0.5, lmd=1.0, low_rank=m + 50)          # clamped to M
    rb = b.registration(tgt, w=0.0, maxiter=4, tol=-1.0)
    assert rb.transformation.q.shape == (m, m)
    # G by MUFU.EX2 on scaled coordinates vs expf: ~3e-7 per entry, amplified by the ill-conditioned solve (4e-6 on the moved
    # points when the emulation perturbs ex2 like MUFU does, CPD_EMU_EX2=mufu)
    assert rb.sigma2 == pytest.approx(ra.sigma2, rel=5e-6)
    np.testing.assert_allclose(b.moved_source(), a.moved_source(), atol=5e-5)


def _check_misc():
    src, tgt = _deformed_pair(200)
    a = cpd.NonRigidCPD(src, low_rank=20, low_rank_seed=3).registration(tgt, maxiter=3, tol=-1.0)
    b = cpd.NonRigidCPD(src, low_rank=20, low_rank_seed=3).registration(tgt, maxiter=3, tol=-1.0)
    assert a.sigma2 == b.sigma2 and np.array_equal(a.transformation.w, b.transformation.w)       # seeded, deterministic
    c = cpd.NonRigidCPD(src, low_rank=20, low_rank_seed=4).registration(tgt, maxiter=3, tol=-1.0)
    assert c.sigma2 == pytest.approx(a.sigma2, rel=1e-4)                   # another basis, (nearly) the same subspace
    seen = []
    r = cpd.registration_cpd(src, tgt, "nonrigid", maxiter=3, tol=-1.0, low_rank=20, callbacks=[lambda t: seen.append(t.w.copy())])
    assert len(seen) == 3 and r.sigma2 == pytest.approx(a.sigma2, rel=1e-4) and not np.array_equal(seen[0], seen[2])
    # one template, several targets: the second registration keeps G / the factors (cpd_nonrigid_restart) and must give exactly
    # what a fresh object gives
    tgt2 = tgt + 0.01
    for kw in ({"low_rank": 20}, {}):
        reuse = cpd.NonRigidCPD(src, **kw)
        reuse.registration(tgt, maxiter=2, tol=-1.0)
        r2 = reuse.registration(tgt2, maxiter=3, tol=-1.0, w=0.1)
        f2 = cpd.NonRigidCPD(src, **kw).registration(tgt2, maxiter=3, tol=-1.0, w=0.1)
        assert r2.sigma2 == f2.sigma2 and np.array_equal(r2.transformation.w, f2.transformation.w)
        src_b = src + 0.5                                                   # ... and an edited source rebuilds them
        reuse.set_source(src_b)
        r3 = reuse.registration(tgt2 + 0.5, maxiter=2, tol=-1.0)
        f3 = cpd.NonRigidCPD(src_b, **kw).registration(tgt2 + 0.5, maxiter=2, tol=-1.0)
        assert r3.sigma2 == f3.sigma2
    # one HANDLE through changing sizes and modes (buffers are re-used / re-allocated inside the library): every run must
    # equal the same run on a fresh handle
    def run_on(h, m, rank):
        s_, t_ = _deformed_pair(m, seed=m)
        h.set_source(s_)
        h.set_target(t_)
        s2 = h.sigma2_init()
        if rank:
            h.nonrigid_lowrank_begin(1.0, 2.0, s2, 0.05, rank, 1, 5)
        else:
            h.nonrigid_begin(1.0, 2.0, s2, 0.05)
        return [h.nonrigid_step() for _ in range(2)], h.nonrigid_w(), h.nonrigid_moved()

    shared = _cabi.Handle(3)
    for m, rank in [(150, 20), (90, 0), (210, 33), (210, 0), (60, 60), (150, 8)]:
        got, want = run_on(shared, m, rank), run_on(_cabi.Handle(3), m, rank)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), (m, rank)
    # default tolerance: stops like the dense loop does (q == sigma2, cpd.py:303)
    d = cpd.NonRigidCPD(src, low_rank=20)
    rd = d.registration(tgt)
    assert 0.0 < rd.sigma2 < a.sigma2
    # 2-D
    s2 = np.random.default_rng(2).random((150, 2))
    t2 = s2 + 0.02 * np.sin(6.0 * s2[:, ::-1])
    r2 = cpd.NonRigidCPD(s2, beta=1.0, lmd=1.0, low_rank=30)
    res2 = r2.registration(t2, maxiter=5, tol=-1.0)
    o2, _ = orc.registration(s2, t2, "nonrigid", maxiter=5, tol=-1.0, beta=1.0, lmd=1.0)
    assert res2.sigma2 == pytest.approx(o2.sigma2, rel=1e-4)
    # argument errors
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    for bad in (0, -3, 5000):
        with pytest.raises(_cabi.CpdError):
            h.nonrigid_lowrank_begin(2.0, 2.0, 0.01, 0.0, bad)
    with pytest.raises(_cabi.CpdError):
        h.nonrigid_lowrank_factors()                                       # nothing begun
    h.nonrigid_begin(2.0, 2.0, 0.01, 0.0)
    with pytest.raises(_cabi.CpdError):
        h.nonrigid_lowrank_factors()                                       # dense mode has no factors
    with pytest.raises(ValueError):
        h.nonrigid_set_prior(1e-2, np.zeros(5), np.zeros((5, 3)))


def _check_standalone_mstep():
    """maximization_step on a caller-supplied EstepResult (cpd.py:284-303 / 376-404): dense, low-rank and constrained."""
    # sigma2 at 2e-6: G is float32 and its entries differ from the reference's in the last bit (expf implementations)
    src, tgt = _deformed_pair(240)
    es = orc.expectation_step(src, tgt, 0.01, 0.05)
    g = orc.rbf_kernel_f32(src, src, 0.7)
    ref = orc.mstep_nonrigid(src, tgt, es, 0.01, g, 1.5)
    reg = cpd.NonRigidCPD(src, beta=0.7, lmd=1.5)
    res = reg.maximization_step(tgt, cpd.EstepResult(*es), 0.01)
    assert res.sigma2 == pytest.approx(ref.sigma2, rel=2e-6) and res.q == res.sigma2
    # (the M x M system is ill-conditioned: another pivot order moves G W by ~1e-6; sigma2 is far more stable)
    np.testing.assert_allclose(reg.moved_source(), src + g.dot(ref.params[0]), atol=1e-5)
    np.testing.assert_allclose(res.transformation.transform(src), src + g.dot(ref.params[0]), atol=2e-5)   # float32 g times an ill-conditioned w
    # a second call with another EstepResult reuses G (source unchanged) ...
    es2 = orc.expectation_step(src, tgt, 0.004, 0.0)
    ref2 = orc.mstep_nonrigid(src, tgt, es2, 0.004, g, 1.5)
    res2 = reg.maximization_step(tgt, cpd.EstepResult(*es2), 0.004)
    assert res2.sigma2 == pytest.approx(ref2.sigma2, rel=2e-6)
    # ... and notices an edited source
    reg.set_source(src * 1.01)
    g3 = orc.rbf_kernel_f32(src * 1.01, src * 1.01, 0.7)
    ref3 = orc.mstep_nonrigid(src * 1.01, tgt, es2, 0.004, g3, 1.5)
    assert reg.maximization_step(tgt, cpd.EstepResult(*es2), 0.004).sigma2 == pytest.approx(ref3.sigma2, rel=2e-6)
    # the reference's static form
    tfo = cpd.tf.NonRigidTransformation(None, src, 0.7)
    st = cpd.NonRigidCPD._maximization_step(src, tgt, cpd.EstepResult(*es), 0.01, tfo, 1.5)
    assert st.sigma2 == pytest.approx(ref.sigma2, rel=2e-6) and st.transformation is tfo and tfo.w.shape == src.shape
    # constrained
    idx = np.arange(0, 240, 9)
    p1t, pxt = orc.constraint_terms(240, tgt, idx, idx)
    refc = orc.mstep_nonrigid(src, tgt, es, 0.01, g, 1.5, alpha=1e-2, p1_tilde=p1t, px_tilde=pxt)
    regc = cpd.ConstrainedNonRigidCPD(src, beta=0.7, lmd=1.5, alpha=1e-2, idx_source=idx, idx_target=idx)
    resc = regc.maximization_step(tgt, cpd.EstepResult(*es), 0.01)
    assert resc.sigma2 == pytest.approx(refc.sigma2, rel=2e-6)
    np.testing.assert_allclose(regc.moved_source(), src + g.dot(refc.params[0]), atol=1e-5)
    # low-rank: against the K x K oracle on the device's own factors
    regl = cpd.NonRigidCPD(src, beta=0.7, lmd=1.5, low_rank=50)
    resl = regl.maximization_step(tgt, cpd.EstepResult(*es), 0.01)
    tfm = resl.transformation
    refl = orc.mstep_nonrigid_lowrank(src, tgt, es, 0.01, tfm.q, tfm.bcore, 1.5)
    assert resl.sigma2 == pytest.approx(refl.sigma2, rel=2e-6)
    np.testing.assert_allclose(regl.moved_source(), refl.params[1], atol=1e-8)
    np.testing.assert_allclose(tfm.w, refl.params[0], atol=1e-6 * np.abs(refl.params[0]).max())


def test_standalone_mstep_emulated(emulated):
    _check_standalone_mstep()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_standalone_mstep_gpu():
    _check_standalone_mstep()


def test_lowrank_vs_oracles_emulated(emulated):
    _check_against_oracles(260, 36, 5, 2.0, 2.0, 0.05, 1e-4)


def test_lowrank_constrained_emulated(emulated):
    _check_against_oracles(220, 32, 4, 1.0, 1.5, 0.0, 1e-4, constrained=True)


def test_lowrank_full_rank_equals_dense_emulated(emulated):
    _check_full_rank_equals_dense(70)


def test_lowrank_misc_emulated(emulated):
    _check_misc()


def test_sliced_dot_products_give_the_same_basis_emulated(emulated, monkeypatch):
    """The Gram-Schmidt dot products are split into up to 8 point slices once M is large; force that at a small M and
    compare with the unsliced run (same arithmetic up to the order of a handful of FP64 additions)."""
    src, tgt = _deformed_pair(300)
    base = cpd.NonRigidCPD(src, low_rank=24).registration(tgt, maxiter=2, tol=-1.0)
    monkeypatch.setenv("CPD_B200_LR_SLICE_POINTS", "48")                      # 300 points -> 7 slices
    sliced = cpd.NonRigidCPD(src, low_rank=24).registration(tgt, maxiter=2, tol=-1.0)
    qb, qs = base.transformation.q, sliced.transformation.q
    np.testing.assert_allclose(qs.T.dot(qs), np.identity(24), atol=1e-12)
    np.testing.assert_allclose(qs.dot(sliced.transformation.bcore).dot(qs.T), qb.dot(base.transformation.bcore).dot(qb.T), atol=2e-6)
    assert sliced.sigma2 == pytest.approx(base.sigma2, rel=1e-6)       # the trailing columns are rounding noise: another summation order, another noise basis


def _check_blocked_orthonormalisation(m, rank):
    """The blocked orthonormalisation (panels of 16 columns, Cholesky inside the panel) against the column-wise one it replaced
    (CPD_B200_LR_ORTH=columnwise), at a rank beyond the numerical rank of G so that columns get dropped and Cholesky pivots get lost:
    same kept / dropped decision per column, orthonormal kept columns, the same G ~= Q Bc Q^T."""
    src, tgt = _deformed_pair(m)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt)
    h.nonrigid_lowrank_begin(2.0, 2.0, 0.05, 0.0, rank, 1, 3)
    qb, bb = h.nonrigid_lowrank_factors()
    os.environ["CPD_B200_LR_ORTH"] = "columnwise"
    try:
        h2 = _cabi.Handle(3)
        h2.set_source(src)
        h2.set_target(tgt)
        h2.nonrigid_lowrank_begin(2.0, 2.0, 0.05, 0.0, rank, 1, 3)
        qc, bc = h2.nonrigid_lowrank_factors()
    finally:
        del os.environ["CPD_B200_LR_ORTH"]
    gram = qb.T.dot(qb)
    d = np.diag(gram)
    assert np.all((np.abs(d - 1.0) < 1e-11) | (d == 0.0))
    np.testing.assert_allclose(gram - np.diag(d), 0.0, atol=1e-11)
    dc = np.diag(qc.T.dot(qc))
    assert abs(int((d == 0).sum()) - int((dc == 0).sum())) <= 1          # a column at the 1e-14 threshold may fall either way
    # the two versions pick different bases for the directions that are float32 noise of G: entries of G ~ 1 agree to that noise
    np.testing.assert_allclose(qb.dot(bb).dot(qb.T), qc.dot(bc).dot(qc.T), atol=5e-6)
    return int((d == 0).sum())


def test_blocked_orthonormalisation_emulated(emulated):
    _check_blocked_orthonormalisation(300, 70)
    _check_blocked_orthonormalisation(150, 150)                           # K = M: every direction, most of them rounding noise


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_blocked_orthonormalisation_gpu():
    _check_blocked_orthonormalisation(3000, 200)
    _check_blocked_orthonormalisation(400, 400)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_vs_oracles_gpu():
    _check_against_oracles(2000, 100, 6, 2.0, 2.0, 0.05, 2e-5)
    _check_against_oracles(1500, 60, 6, 0.3, 1.5, 0.0, 1e-3)               # narrow kernel: slower spectral decay


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_constrained_gpu():
    _check_against_oracles(1500, 80, 5, 1.0, 1.5, 0.0, 5e-5, constrained=True)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_full_rank_equals_dense_gpu():
    _check_full_rank_equals_dense(400)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_misc_gpu():
    _check_misc()


def _check_spd_core(m, rank, iters, monkeypatch, noise_level=False):
    """By default the M-step solves the symmetric positive definite system of the factor Qt = Q L, Bc ~= L L^T (pivoted Cholesky at
    set-up, one-CTA LDL^T per iteration); CPD_B200_LR_CORE=lu keeps the unsymmetric (c I + Bc S) Z = Bc R and its LU (also what ranks
    above LR_SPD_MAX_RANK = 232 use).  Same Q and Bc, same registration, up to the rounding of two different solves.  `noise_level`:
    the rank reaches into the float32 noise of the G X products (K ~ M), where Bc has eigenvalues of both signs at the 1e-7 level;
    the Cholesky factor stops there (G is positive semi-definite), the LU keeps them -- the tolerance is then that noise."""
    src, tgt = _deformed_pair(m)
    spd = cpd.NonRigidCPD(src, beta=1.5, lmd=2.0, low_rank=rank)
    rs = spd.registration(tgt, w=0.05, maxiter=iters, tol=-1.0)
    monkeypatch.setenv("CPD_B200_LR_CORE", "lu")
    lu = cpd.NonRigidCPD(src, beta=1.5, lmd=2.0, low_rank=rank)
    rl = lu.registration(tgt, w=0.05, maxiter=iters, tol=-1.0)
    monkeypatch.delenv("CPD_B200_LR_CORE")
    ts, tl = rs.transformation, rl.transformation
    assert np.array_equal(ts.q, tl.q)
    # the exported core is L L^T in the default form, the raw Q^T G Q with the LU: they differ by what the Cholesky factor left out
    np.testing.assert_allclose(ts.bcore, tl.bcore, atol=(2e-6 if noise_level else 1e-8) * np.abs(tl.bcore).max())
    if rank <= 232:
        assert np.linalg.eigvalsh(ts.bcore).min() > -1e-12 * np.abs(ts.bcore).max()             # positive semi-definite
    assert rs.sigma2 == pytest.approx(rl.sigma2, rel=1e-5 if noise_level else 1e-7)
    np.testing.assert_allclose(spd.moved_source(), lu.moved_source(), atol=1e-4 if noise_level else 1e-6)
    np.testing.assert_allclose(ts.w, tl.w, atol=(1e-2 if noise_level else 2e-5) * max(1.0, np.abs(tl.w).max()))   # W = (...) / (lmd sigma2): the least stable output
    np.testing.assert_allclose(ts.transform(src), spd.moved_source(), atol=1e-4 if noise_level else 1e-8)


def test_spd_core_equals_lu_core_emulated(emulated, monkeypatch):
    _check_spd_core(260, 36, 4, monkeypatch)
    _check_spd_core(120, 120, 3, monkeypatch, noise_level=True)          # K = M: dropped columns, pivoted Cholesky stops early
    _check_spd_core(300, 240, 2, monkeypatch, noise_level=True)          # above LR_SPD_MAX_RANK: both runs take the LU


def test_spd_core_at_tiny_and_ragged_ranks_emulated(emulated, monkeypatch):
    """Ranks below, at and just above the panel width of the blocked LDL^T (8), and one that is no multiple of it."""
    for rank in (1, 2, 7, 8, 9, 17):
        _check_spd_core(90, rank, 2, monkeypatch)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_spd_core_at_tiny_and_ragged_ranks_gpu(monkeypatch):
    for rank in (1, 7, 8, 9, 63, 228):
        _check_spd_core(1200, rank, 2, monkeypatch, noise_level=rank > 20)     # 63 of 1200 points already reaches the float32 noise


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_spd_core_equals_lu_core_gpu(monkeypatch):
    _check_spd_core(3000, 40, 6, monkeypatch)
    _check_spd_core(3000, 200, 6, monkeypatch, noise_level=True)
    _check_spd_core(300, 300, 3, monkeypatch, noise_level=True)
    _check_spd_core(1000, 240, 3, monkeypatch, noise_level=True)


def _check_config5(m_cross, m_big, rank, iters):
    """BASELINE configuration 5 (N = M = 50k, K = 200): size-independent properties, and the dense device loop at a size it
    can still afford as the cross-check."""
    src, tgt = _deformed_pair(m_cross)
    a = cpd.NonRigidCPD(src, beta=2.0, lmd=2.0)
    ra = a.registration(tgt, maxiter=5, tol=-1.0)
    b = cpd.NonRigidCPD(src, beta=2.0, lmd=2.0, low_rank=rank)
    rb = b.registration(tgt, maxiter=5, tol=-1.0)
    assert rb.sigma2 == pytest.approx(ra.sigma2, rel=5e-5)              # emulation with a MUFU-like ex2 at 6k: 1.2e-5 / 5.1e-5
    np.testing.assert_allclose(b.moved_source(), a.moved_source(), atol=2e-4)
    src, tgt = _deformed_pair(m_big)
    trace = []
    reg = cpd.NonRigidCPD(src, beta=2.0, lmd=2.0, low_rank=rank)
    reg.set_callbacks([lambda t: trace.append(t.w is not None)])
    res = reg.registration(tgt, maxiter=iters, tol=-1.0)
    assert len(trace) == iters and all(trace)
    q = res.transformation.q
    assert q.shape == (m_big, min(rank, m_big))
    gram = q.T.dot(q)
    d = np.diag(gram)
    assert np.all((np.abs(d - 1.0) < 1e-11) | (d == 0.0))
    moved = reg.moved_source()
    assert np.isfinite(moved).all() and np.isfinite(res.sigma2) and res.sigma2 > 0
    # the deformation is recovered: residual to the (unpermuted) target well below the 0.03 amplitude that was applied.  Non-rigid
    # CPD first SHRINKS the cloud while sigma2 is large (after 8-10 iterations the residual has doubled) and needs ~30 to come back
    assert np.sqrt(((moved - tgt) ** 2).sum(1)).mean() < 0.4 * np.sqrt(((src - tgt) ** 2).sum(1)).mean()


def test_config5_body_at_emulation_size(emulated):
    _check_config5(260, 500, 40, 40)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_baseline_config5_properties():
    _check_config5(6000, 50000, 200, 80)      # residual 0.26 of the applied deformation after 80 iterations (0.43 after 60;
                                                # the dense loop at 12k follows the same curve)


_PRODUCT_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, %r)
from oracle import cpd_oracle as orc
from probreg_b200 import _cabi
src, _ = orc.synthetic_pair(%d)
h = _cabi.Handle(3)
h.set_source(src)
h.set_target(src[:64] + 0.01)
h.nonrigid_lowrank_begin(%g, 2.0, 0.05, 0.0, %d, 1, 5)
q, b = h.nonrigid_lowrank_factors()
np.save(sys.argv[1], q.dot(b).dot(q.T))
"""


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_every_selectable_gram_product_gives_the_same_factorisation(tmp_path):
    """CPD_B200_LR_GRAM selects the kernel behind the G X products of the range finder: the exact integer-digit tensor-core kernel
    (the default) or the CUDA-core kernel.  The variable is read once per process, hence subprocesses.  Both agree with the float32
    G of the reference to 1e-6 (relative, spectral norm).  A rank of 130 takes three column passes, 1300 points 11 row tiles."""
    import subprocess
    import sys

    from conftest import ROOT

    m, rank, beta = 1300, 130, 0.6
    src, _ = orc.synthetic_pair(m)
    g = orc.rbf_kernel_f32(src, src, beta).astype(np.float64)
    code = _PRODUCT_SCRIPT % (ROOT, m, beta, rank)
    errs = {}
    for mode in ("i8", "simt"):
        out = str(tmp_path / ("g_%s.npy" % mode))
        r = subprocess.run([sys.executable, "-c", code, out], capture_output=True, text=True, timeout=600,
                           env=dict(os.environ, CPD_B200_LR_GRAM=mode))
        assert r.returncode == 0, (mode, r.stderr[-2000:])
        errs[mode] = np.linalg.norm(np.load(out) - g, 2) / np.linalg.norm(g, 2)
    assert errs["i8"] < 1e-6 and errs["simt"] < 1e-6, errs
