"""oracle/sparse_oracle.py against the dense float64 oracle (no GPU, no emulation): the neighbour-search E-steps must be the
reference's E-steps, so that the full-size tests (test_zz_estep_fullsize.py) can compare the kernels with them element-wise."""
import numpy as np
import pytest

from oracle import cpd_oracle as orc
from oracle import sparse_oracle as so

TOL = 1e-13


def _cloud(n, dim, seed, kind):
    rng = np.random.default_rng(seed)
    src = rng.random((n, dim)) * np.array([1.0, 0.6, 0.3])[:dim]
    tgt = src[rng.permutation(n)] + 0.01 * rng.standard_normal((n, dim))
    if kind == "dup":                              # duplicated sources, targets exactly on sources, far outliers
        src[1::7] = src[0::7][: len(src[1::7])]
        tgt[::5] = src[::5][: len(tgt[::5])]
        tgt[-20:] += 50.0
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt)


def _same(got, ref, tol=TOL):
    np.testing.assert_array_equal(got.pt1 == 0, ref.pt1 == 0)
    for g, r in ((got.pt1, ref.pt1), (got.p1, ref.p1), (got.px, ref.px)):
        np.testing.assert_allclose(g, r, rtol=tol, atol=tol * max(1e-300, np.abs(r).max()))


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("s2", [1e-7, 1e-5, 1e-3, 1e-1, 1.0])
@pytest.mark.parametrize("w", [0.0, 0.1, 0.5])
def test_estep_equals_dense_oracle(dim, s2, w):
    src, tgt = _cloud(2500, dim, 1, "plain")
    got = so.expectation_step(src, tgt, s2, w, chunk=700)
    ref = orc.expectation_step(src, tgt, s2, w)
    _same(got.es, ref)
    assert got.es.n_p == pytest.approx(ref.n_p, rel=TOL, abs=1e-300)


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("s2", [1e-6, 1e-4])
def test_estep_duplicates_coincidences_outliers_and_a_shard(dim, s2):
    src, tgt = _cloud(3000, dim, 2, "dup")
    for w, ng in ((0.0, None), (0.1, None), (0.1, 24000)):
        got = so.expectation_step(src, tgt, s2, w, n_global=ng)
        ref = orc.expectation_step(src, tgt, s2, w, n_global=ng)
        _same(got.es, ref)
        assert (ref.pt1 == 0).sum() >= 20                    # the far outliers' columns are dead, identically


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("s2", [1e-6, 1e-4, 1e-2])
@pytest.mark.parametrize("w", [0.0, 0.1, 0.5])
def test_bcpd_estep_equals_dense_oracle(dim, s2, w):
    src, tgt = _cloud(1500, dim, 3, "dup")
    rng = np.random.default_rng(4)
    alpha = rng.dirichlet(np.full(len(src), 0.5))
    sdiag = rng.uniform(0.0, 3.0 * s2, len(src))
    got = so.bcpd_expectation_step(src, tgt, 1.1, alpha, sdiag, s2, w, chunk=400)
    ref = orc.bcpd_expectation_step(src, tgt, 1.1, alpha, sdiag, s2, w)
    for g, r in ((got.es.pt1, ref.nu_d), (got.es.p1, ref.nu), (got.es.px, ref.px)):
        np.testing.assert_allclose(g, r, rtol=TOL, atol=TOL * max(1e-300, np.abs(r).max()))


def test_a_source_exactly_at_the_cut_radius_is_kept_and_one_beyond_it_is_not():
    """One target at the origin, its nearest source at u = 1 (log2 units), one source at exactly u = 1 + R, one beyond."""
    s2 = 0.5 * so.LOG2E                                       # f = LOG2E / (2 s2) = 1: u = |d|^2
    r_cut = np.sqrt(1.0 + so.R_LOG2)
    src = np.array([[1.0, 0.0, 0.0], [0.0, r_cut, 0.0], [0.0, 0.0, r_cut * (1.0 + 1e-6)]])
    assert ((src[1] ** 2).sum()) == 1.0 + so.R_LOG2           # exactly representable: the cut itself
    tgt = np.zeros((1, 3))
    got = so.expectation_step(src, tgt, s2, 0.0)
    assert got.extras.pairs == 2 and got.extras.row_cnt.tolist() == [1, 1, 0]
    assert got.es.p1[1] == pytest.approx(2.0 ** -so.R_LOG2, rel=1e-15)          # 2^-(1 + R) / 2^-1
    assert got.es.p1[2] == 0.0


def test_the_cut_is_exact_for_float64():
    """Everything beyond the cut is below 2^-160 of the column's largest term: the dense oracle sees no difference."""
    src, tgt = _cloud(2000, 3, 5, "plain")
    s2 = 3e-4                                                 # many sources beyond u_nn + R for every column
    got = so.expectation_step(src, tgt, s2, 0.0)
    assert got.extras.pairs < 0.9 * src.shape[0] * tgt.shape[0]
    _same(got.es, orc.expectation_step(src, tgt, s2, 0.0), tol=1e-14)


def test_denormal_band_columns_are_reported():
    src = np.zeros((1, 3))
    s2 = 1e-4
    d = np.sqrt(2.0 * s2 * np.array([100.0, 700.0, 750.0, 800.0]))   # d^2 / 2 s2 in natural units
    tgt = np.c_[d, np.zeros(4), np.zeros(4)]
    got = so.expectation_step(src, tgt, s2, 0.0)
    assert got.extras.band.tolist() == [False, True, True, False]


def test_rounded_mode_reproduces_pack_kernel_on_a_hand_case():
    """pack_kernel: a = fl32(sk (p - c_x)) with sk = sqrt(LOG2E / (2 s2)) in FP64.  At s2 = LOG2E / 2, sk = 1 exactly: the
    float32 roundings of the differences can be written out by hand."""
    s2 = so.LOG2E / 2.0
    assert np.sqrt(so.LOG2E / (2.0 * s2)) == 1.0
    org = np.array([0.5, -0.25, 1.0])
    pts = np.array([[0.5 + 2.0 ** -30, 1.0 / 3.0, 1.0 + 2.0 ** -24 + 2.0 ** -50]])
    a = so.pack_coordinates(pts, s2, org)
    third = 1.0 / 3.0 + 0.25                                  # 0.58333...: float32 0x3F155555 = 9786709 * 2^-24
    assert a[0, 0] == 2.0 ** -30                              # exact
    assert a[0, 1] == 9786709.0 * 2.0 ** -24 and abs(a[0, 1] - third) < 2.0 ** -25
    assert a[0, 2] == 2.0 ** -24                              # 2^-24 (1 + 2^-26) rounds to 2^-24
    # sigma2 = 1e-6: sk * 0.1 = 84.932180028801..., whose float32 neighbours are k * 2^-17: k = 11132231 (84.93218231...)
    b = so.pack_coordinates(np.array([[0.1, 0.0, 0.0]]), 1e-6, np.zeros(3))
    assert b[0, 0] == 11132231.0 * 2.0 ** -17 and b[0, 1] == 0.0


@pytest.mark.parametrize("dim", [2, 3])
def test_rounded_mode_with_large_sigma_equals_the_unrounded_mode(dim):
    """With sigma ~ extent the FP32 rounding of the sigma-scaled coordinates moves u by ~2^-24 |a| |a - b| only: both modes
    agree to that bound, and px is the same sum written two ways."""
    src, tgt = _cloud(1500, dim, 6, "plain")
    org = tgt.mean(0)
    for s2, w in ((0.5, 0.0), (0.05, 0.1)):
        plain = so.expectation_step(src, tgt, s2, w)
        rnd = so.expectation_step(src, tgt, s2, w, frame_origin=org)
        sk = np.sqrt(so.LOG2E / (2.0 * s2))
        ext = sk * max(np.abs(src - org).max(), np.abs(tgt - org).max())
        du = 4.0 * 2.0 ** -24 * ext * (2.0 * ext) * dim        # |delta u| <= sum_i 2 |a_i - b_i| (|da_i| + |db_i|)
        rel = 3.0 * du * np.log(2.0)                          # K, and the column sum and the other terms of P
        np.testing.assert_allclose(rnd.es.pt1, plain.es.pt1, rtol=rel, atol=0)
        np.testing.assert_allclose(rnd.es.p1, plain.es.p1, rtol=rel, atol=0)
        np.testing.assert_allclose(rnd.es.px, plain.es.px, rtol=rel, atol=rel * np.abs(plain.es.px).max())
        assert np.abs(rnd.es.p1 / plain.es.p1 - 1.0).max() > 1e-12          # ... and the rounding is really there


def test_bound_sums_on_a_two_source_column():
    """The per-element sums the bound is made of, on a column with two sources at u = 0 and u = 1 (log2 units)."""
    s2 = 0.5 * so.LOG2E
    src = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])
    got = so.expectation_step(src, np.zeros((1, 3)), s2, 0.0)
    p = np.array([2.0 / 3.0, 1.0 / 3.0])                      # 2^0 / 1.5, 2^-1 / 1.5
    np.testing.assert_allclose(got.es.p1, p, rtol=1e-15)
    np.testing.assert_allclose(got.extras.col_dbar, [p[1] * 1.0], rtol=1e-15)       # K-weighted mean of u
    np.testing.assert_allclose(got.extras.row_pd, [0.0, p[1]], rtol=1e-15)
    np.testing.assert_allclose(got.extras.row_pdbar, p * p[1], rtol=1e-15)
    assert got.extras.row_cnt.tolist() == [1, 1] and got.extras.col_cnt.tolist() == [2] and got.extras.col_umin[0] == 0.0
