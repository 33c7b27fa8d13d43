"""SVR (cpd_ocsvm_fit; probreg_b200.features.OneClassSVM, l2dist_regs.RigidSVR / TPSSVR / registration_svr).

  1. the oracle (oracle/ocsvm_oracle.py) against sklearn's OneClassSVM: identical n_iter_, alpha bit-identical, equal support and
     intercept_; a far-translated cloud to a tolerance;
  2. the oracle's registrations against the reference's (tests/golden/svr.npz, made by make_golden_svr.py), with the fixture's
     features replayed and with the oracle's own;
  3. cpd_ocsvm_fit against the oracle: n_iter, support, alpha, rho; two runs bit-identical; the refusals;
  4. the Python surface: registration_svr rigid and nonrigid with device features against svr.npz;
  5. (GPU) 100 000 and 1 000 000 points: the constraints, a bit-identical rerun, the KKT gap checked through cpd_gauss_transform,
     the device memory the fit takes.
CPU tests run under the emulation of tests/emu at small sizes; the gpu-marked ones on the H100.
"""
import numpy as np
import pytest

from conftest import load_golden
from oracle import l2dist_oracle as lo
from oracle import ocsvm_oracle as oo
from probreg_b200 import _cabi, features, gauss_transform, l2dist_regs, transformation


def _rot(axis, deg):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.identity(3) + np.sin(th) * k + (1.0 - np.cos(th)) * k.dot(k)


def _bunny():
    return np.ascontiguousarray(load_golden("bunny.npz")["source"])


def _fish():
    import os

    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
    return np.loadtxt(os.path.join(d, "fish_source.txt")), np.loadtxt(os.path.join(d, "fish_target.txt"))


def _box(n, seed=0):
    return np.random.default_rng(seed).random((n, 3)) * [1.0, 0.6, 0.3]


def _gamma(x, factor=1.0):
    return factor / (2.0 * lo.estimate_sigma(x) ** 2)


def _cloud(name):
    """(points, nu, gamma) of a named case"""
    b = _bunny()
    return {
        "bunny": lambda: (b, 0.1, _gamma(b)),
        "bunny_g10": lambda: (b, 0.1, _gamma(b, 10.0)),
        "bunny_g100": lambda: (b, 0.1, _gamma(b, 100.0)),
        "fish": lambda: (_fish()[0], 0.1, _gamma(_fish()[0])),
        "box5k": lambda: (_box(5000), 0.1, _gamma(_box(5000))),
        "dup": lambda: (np.vstack([b, b[:50]]), 0.1, _gamma(np.vstack([b, b[:50]]))),
        "2d": lambda: (b[:700, :2].copy(), 0.1, _gamma(b[:700, :2])),
        "nul_integral": lambda: (b[:400], 0.25, _gamma(b[:400])),           # nu l = 100
        "nul_below_1": lambda: (b[:600], 0.5 / 600, _gamma(b[:600])),       # a single start alpha of 0.5
        "box300": lambda: (_box(300, 3), 0.3, _gamma(_box(300, 3), 3.0)),
    }[name]()


def _full(clf, n):
    a = np.zeros(n)
    a[clf.support_] = clf.dual_coef_[0]
    return a


# ---- 1. the oracle against sklearn ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["bunny", "bunny_g10", "bunny_g100", "fish", "box5k", "dup", "2d", "nul_integral", "nul_below_1"])
def test_oracle_matches_sklearn(name):
    svm = pytest.importorskip("sklearn.svm")
    x, nu, g = _cloud(name)
    a, rho, it, _ = oo.fit(x, nu, g)
    # bit-identical to the unshrunk solver; sklearn's default shrinking rebuilds G, which moves alpha by at most ~1e-14
    for shrinking, atol in ((False, 0.0), (True, 1e-13)):
        ref = svm.OneClassSVM(nu=nu, kernel="rbf", gamma=g, shrinking=shrinking).fit(x)
        assert it == int(ref.n_iter_)
        assert np.abs(a - _full(ref, len(x))).max() <= atol
        np.testing.assert_array_equal(np.nonzero(a > 0)[0], ref.support_)
        assert abs(-rho - ref.intercept_[0]) <= 1e-12 * abs(rho)


def test_oracle_nu_one_and_sklearn_refuses():
    svm = pytest.importorskip("sklearn.svm")
    x = _bunny()[:300]
    a, rho, it, _ = oo.fit(x, 1.0, _gamma(x))
    assert it == 0 and (a == 1.0).all() and rho == np.inf
    with pytest.raises(ValueError, match="not finite"):
        svm.OneClassSVM(nu=1.0, kernel="rbf", gamma=_gamma(x)).fit(x)


def test_oracle_matches_sklearn_with_shrinking_20k():
    """sklearn's default shrinking acts at 20 000 points and leaves the path of the unshrunk solver"""
    svm = pytest.importorskip("sklearn.svm")
    x = _box(20_000, 1)
    g = _gamma(x)
    ref = svm.OneClassSVM(nu=0.1, kernel="rbf", gamma=g, shrinking=True).fit(x)
    a, rho, it, _ = oo.fit(x, 0.1, g)
    assert it == int(ref.n_iter_)
    assert np.abs(a - _full(ref, len(x))).max() <= 1e-13
    assert abs(-rho - ref.intercept_[0]) <= 1e-12 * abs(rho)


def test_oracle_far_from_origin_to_a_tolerance():
    """|x|^2 + |y|^2 - 2 x.y cancels far from the origin and rounds differently: the same iterations, alpha to 1e-6"""
    svm = pytest.importorskip("sklearn.svm")
    x = _bunny() + [100.0, -50.0, 20.0]
    g = _gamma(x)
    ref = svm.OneClassSVM(nu=0.1, kernel="rbf", gamma=g).fit(x)
    a, rho, it, _ = oo.fit(x, 0.1, g)
    assert it == int(ref.n_iter_)
    assert np.abs(a - _full(ref, len(x))).max() <= 1e-6
    assert abs(-rho - ref.intercept_[0]) <= 1e-6 * abs(rho)


# ---- 2. the oracle's registrations against the reference's ---------------------------------------------------------------------
def _golden():
    return load_golden("svr.npz")


def _calls(g, pre):
    return [(g["%s%d_sv" % (pre, k)], g["%s%d_w" % (pre, k)]) for k in range(int(g[pre + "n_calls"]))]


def _replayer(feats):
    it = iter(feats)
    return lambda data, gamma: next(it)


def test_oracle_matches_reference_registrations():
    g = _golden()
    bunny = _bunny()
    sigma = lo.estimate_sigma(bunny)
    assert abs(sigma - float(g["bunny_sigma"])) <= 1e-14 * sigma
    for maxiter in (1, 2):
        pre = "bunny%d_" % maxiter
        for feats in (_replayer(_calls(g, pre)), None):
            x = oo.registration(lo.rigid_cost, np.r_[1.0, np.zeros(6)], bunny, g["bunny_target"], sigma, 1.0 / (2.0 * sigma ** 2),
                                maxiter=maxiter, features=feats)
            np.testing.assert_allclose(lo.quat2mat(x[:4]), g[pre + "rot"], rtol=0, atol=1e-8)
            np.testing.assert_allclose(x[4:7], g[pre + "t"], rtol=0, atol=1e-8)
    fs, ft_ = _fish()
    sigma = lo.estimate_sigma(fs)
    calls = _calls(g, "fish_")
    cost = lo.TPSCost(calls[0][0])
    for feats in (_replayer(calls[1:]), None):
        x = oo.registration(cost, cost.initial(), fs, ft_, sigma, 1.0 / (2.0 * sigma ** 2), features=feats)
        a, v = cost.split(x)
        assert np.abs(a - g["fish_a"]).max() <= 1e-8 * np.abs(g["fish_a"]).max()
        assert np.abs(v - g["fish_v"]).max() <= 1e-8 * np.abs(g["fish_v"]).max()


def test_reference_recovers_most_of_ten_degrees():
    g = _golden()
    ang = np.rad2deg(np.arccos((np.trace(g["bunny1_rot"]) - 1.0) / 2.0))
    assert 8.9 <= ang <= 9.0, ang


# ---- 3. cpd_ocsvm_fit against the oracle ---------------------------------------------------------------------------------------
def _check_fit(x, nu, g, atol, twice=True):
    a, rho, it = _cabi.ocsvm_fit(x, nu, g)
    oa, orho, oit, _ = oo.fit(x, nu, g)
    assert it == oit
    np.testing.assert_array_equal(a > 0, oa > 0)
    assert np.abs(a - oa).max() <= atol, np.abs(a - oa).max()
    if np.isfinite(orho):
        assert abs(rho - orho) <= 1e-12 * abs(orho)
    else:
        assert rho == orho
    if twice:
        a2, rho2, it2 = _cabi.ocsvm_fit(x, nu, g)
        np.testing.assert_array_equal(a, a2)
        assert rho2 == rho and it2 == it
    print("ocsvm n=%d nu=%g: %d iterations, %d support vectors, max |da| %.3g" % (len(x), nu, it, (a > 0).sum(), np.abs(a - oa).max()))


EMU_CASES = ["bunny", "fish", "dup", "2d", "nul_integral", "nul_below_1", "box300"]


@pytest.mark.parametrize("name", EMU_CASES)
def test_fit_matches_oracle_emulated(emulated, name):
    _check_fit(*_cloud(name), atol=1e-12)


def test_fit_edges_emulated(emulated):
    b = _bunny()
    _check_fit(b[:300], 1.0, _gamma(b[:300]), 0.0, twice=False)        # every alpha at 1: no iteration, rho = inf
    _check_fit(b[:1], 0.5, 1.0, 0.0, twice=False)                      # one point
    _check_fit(b[:200] + [100.0, -50.0, 20.0], 0.1, _gamma(b[:200]), 1e-12, twice=False)
    a, rho, it = _cabi.ocsvm_fit(b[:500], 0.1, _gamma(b[:500]), max_iter=7)   # the cap: the iterate after 7 updates
    oa, _, oit, _ = oo.fit(b[:500], 0.1, _gamma(b[:500]), max_iter=7)
    assert it == oit == 7
    np.testing.assert_array_equal(a, oa)


def _check_refusals():
    x = _bunny()[:50]
    for kw, pat in (({"x": x[:, :1]}, "dim"), ({"x": np.zeros((0, 3))}, "at least one point"), ({"nu": 0.0}, "nu"), ({"nu": 1.5}, "nu"),
                    ({"gamma": 0.0}, "gamma"), ({"gamma": np.inf}, "gamma"), ({"tol": 0.0}, "tol"), ({"tol": np.nan}, "tol"),
                    ({"max_iter": 0}, "max_iter")):
        args = dict(x=x, nu=0.1, gamma=1.0)
        args.update(kw)
        with pytest.raises(_cabi.CpdError, match=pat):
            _cabi.ocsvm_fit(**args)
    xb = x.copy()
    xb[7, 1] = np.nan
    with pytest.raises(_cabi.CpdError, match="non-finite"):
        _cabi.ocsvm_fit(xb, 0.1, 1.0)


def test_refusals_emulated(emulated):
    _check_refusals()


# ---- 4. the Python surface -----------------------------------------------------------------------------------------------------
def _check_registrations(maxiters=(1, 2)):
    g = _golden()
    bunny = _bunny()
    for maxiter in maxiters:
        pre = "bunny%d_" % maxiter
        seen = []
        res = l2dist_regs.registration_svr(bunny, g["bunny_target"], maxiter=maxiter, callbacks=[seen.append])
        assert seen and isinstance(res, transformation.RigidTransformation)
        np.testing.assert_allclose(res.rot, g[pre + "rot"], rtol=0, atol=1e-6)
        np.testing.assert_allclose(res.t, g[pre + "t"], rtol=0, atol=1e-6)
        if maxiter == 1:                       # the reference's single outer iteration recovers 8.95 of the 10 degrees
            assert 8.9 <= np.rad2deg(np.arccos((np.trace(res.rot) - 1.0) / 2.0)) <= 9.0
    fs, ft_ = _fish()
    reg = l2dist_regs.TPSSVR(fs)
    np.testing.assert_array_equal(reg._cost_fn._control_pts, g["fish_0_sv"])
    res = reg.registration(ft_)
    assert isinstance(res, transformation.TPSTransformation)
    assert np.abs(res.a - g["fish_a"]).max() <= 1e-6 * np.abs(g["fish_a"]).max()
    assert np.abs(res.v - g["fish_v"]).max() <= 1e-6 * np.abs(g["fish_v"]).max()


def _check_surface():
    b = _bunny()
    oc = features.OneClassSVM(3, 0.05, gamma=_gamma(b), nu=0.1)
    oc.init()
    sv, w = oc(b)
    a, rho, it, _ = oo.fit(b, 0.1, _gamma(b))
    np.testing.assert_array_equal(oc.support_, np.nonzero(a > 0)[0])
    np.testing.assert_array_equal(sv, b[oc.support_])
    assert oc.dual_coef_.shape == (1, len(oc.support_)) and oc.n_iter_ == it
    np.testing.assert_allclose(w, oc.dual_coef_[0] * (2.0 * np.pi * 0.05 ** 2) ** 1.5, rtol=1e-15)
    assert oc.intercept_[0] == -oc.offset_[0] and abs(oc.offset_[0] - rho) <= 1e-12 * rho
    g0 = oc._gamma
    oc.annealing()
    assert oc._gamma == g0 * 10.0
    with pytest.raises(ValueError, match="not finite"):
        features.OneClassSVM(3, 0.05, gamma=1.0, nu=1.0)(b[:40])
    with pytest.warns(features.ConvergenceWarning):
        features.OneClassSVM(3, 0.05, gamma=_gamma(b), nu=0.1, max_iter=5)(b[:300])
    with pytest.raises(ValueError, match="Unknown transform type"):
        l2dist_regs.registration_svr(b, b, tf_type_name="affine")
    reg = l2dist_regs.RigidSVR(b)
    assert reg._feature_gen._sigma == reg._sigma and reg._feature_gen._gamma == 1.0 / (2.0 * reg._sigma ** 2)
    for name in ("RigidSVR", "TPSSVR", "registration_svr"):
        assert hasattr(l2dist_regs, name)


def test_registrations_emulated(emulated):
    _check_registrations(maxiters=(1,))


def test_python_surface_emulated(emulated):
    _check_surface()


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_small_cases_gpu():
    for name in EMU_CASES + ["bunny_g10", "box5k"]:
        _check_fit(*_cloud(name), atol=1e-9)
    x = _box(20_000, 1)
    _check_fit(x, 0.1, _gamma(x), atol=1e-9)
    _check_refusals()
    _check_surface()


@pytest.mark.gpu
def test_registrations_gpu():
    _check_registrations()


def _lumps(n, seed):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-1.0, 1.0, (6, 3))
    scales = rng.uniform(0.05, 0.3, (6, 3))
    lab = rng.integers(0, 6, n)
    return centres[lab] + rng.standard_normal((n, 3)) * scales[lab]


def _check_scale(n, seed, tol=1e-3):
    import time

    import torch

    x = _lumps(n, seed)
    g = _gamma(x)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    t0 = time.perf_counter()
    a, rho, it = _cabi.ocsvm_fit(x, 0.1, g, tol)
    dt = time.perf_counter() - t0
    a2, rho2, it2 = _cabi.ocsvm_fit(x, 0.1, g, tol)
    np.testing.assert_array_equal(a, a2)
    assert rho == rho2 and it == it2
    assert (a >= 0.0).all() and (a <= 1.0).all()
    assert abs(a.sum() - 0.1 * n) <= 1e-9 * 0.1 * n
    # the KKT gap on G = Q alpha formed independently (exact FP64 kernel), with slack for the float32 kernel columns
    sv = np.nonzero(a > 0)[0]
    G = gauss_transform.GaussTransform(x[sv], g ** -0.5).compute(x, a[sv])
    gap = np.max(-G[a < 1.0]) + np.max(G[a > 0.0])
    assert gap <= tol + 2.0 ** -23 * a.sum(), gap
    # the fit's own buffers: x, the points {x, |x|^2}, alpha, G, the float column (76 bytes per point in 3-D) and O(CTAs)
    need = n * (24 + 32 + 8 + 8 + 4)
    print("ocsvm %d points, nu 0.1: %d iterations, %d support vectors, %.3f s, KKT gap %.3g, buffers %.1f MB (free before %.0f MB)"
          % (n, it, len(sv), dt, gap, need / 2 ** 20, free0 / 2 ** 20))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_fit_100k_gpu():
    _check_scale(100_000, 30)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_fit_1m_gpu():
    _check_scale(1_000_000, 31)
