"""GMMReg (cpd_gmm_fit, cpd_l2_dist, cpd_tps_kernel; probreg_b200.features / cost_functions / l2dist_regs).

  1. the oracle (oracle/l2dist_oracle.py) against sklearn's GaussianMixture and against the reference's own outputs
     (tests/golden/l2dist.npz, made by make_golden_l2dist.py);
  2. the oracle's gradients against central differences of f;
  3. cpd_gmm_fit against the oracle: iteration count, parameters, the lower bound per iteration; two runs bit-identical;
  4. cpd_l2_dist against the oracle; 5. cpd_tps_kernel bit-identical to the float32 restatement;
  6. the registrations with the reference's features replayed, against the reference and against the oracle's loop;
  7. a known answer (the bunny under 30 degrees and a translation); 8. the refusals and the Python surface;
  9. (GPU) 100k points x 800 components, 1M points x 800 (bit-identical, EM monotone, memory), the L2 distance at 10 000 x 12 000.
CPU tests run under the emulation of tests/emu at small sizes; the gpu-marked ones on the H100.
"""
import numpy as np
import pytest

from conftest import load_golden
from oracle import l2dist_oracle as lo
from probreg_b200 import _cabi, cost_functions, features, l2dist_regs, math_utils, se3_op, transformation

REL = 1e-9


def _rot(axis, deg):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.identity(3) + np.sin(th) * k + (1.0 - np.cos(th)) * k.dot(k)


def _lumps(n, dim=3, seed=0):
    """a few Gaussian lumps of different widths"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-1.0, 1.0, (6, dim))
    scales = rng.uniform(0.03, 0.3, (6, dim))
    lab = rng.integers(0, 6, n)
    return centres[lab] + rng.standard_normal((n, dim)) * scales[lab]


def _bunny():
    return np.ascontiguousarray(load_golden("bunny.npz")["source"])


def _golden():
    return load_golden("l2dist.npz")


# ---- 1. the oracle against sklearn and the reference ------------------------------------------------------------------------------
def _gauss(n, seed):
    return np.random.default_rng(seed).standard_normal((n, 3)) * [1.0, 0.5, 0.2]


@pytest.mark.parametrize("k,seed,cloud", [(50, 0, "lumps"), (200, 3, "gauss"), (30, 7, "lumps2d")])
def test_oracle_matches_sklearn(k, seed, cloud):
    mixture = pytest.importorskip("sklearn.mixture")
    x = {"lumps": lambda: _lumps(2000, 3, seed), "lumps2d": lambda: _lumps(2000, 2, seed), "gauss": lambda: _gauss(3000, seed)}[cloud]()
    x = np.vstack([x, x[:60]])                 # duplicate points
    ref = mixture.GaussianMixture(k, covariance_type="spherical", init_params="random_from_data", random_state=seed).fit(x)
    w, mu, var, it, lb = lo.gmm_fit(x, k, seed, chunk=700)
    assert it == ref.n_iter_
    for a, b in ((w, ref.weights_), (mu, ref.means_), (var, ref.covariances_)):
        assert np.abs(a - b).max() <= 1e-10 * np.abs(b).max()
    assert abs(lb[-1] - ref.lower_bound_) <= 1e-10 * abs(ref.lower_bound_)


def test_oracle_matches_reference_costs():
    g = _golden()
    for th, f, gr in zip(g["rigid_thetas"], g["rigid_f"], g["rigid_grad"]):
        of, og = lo.rigid_cost(th, g["rigid_ms"], g["rigid_ps"], g["rigid_mt"], g["rigid_pt"], float(g["rigid_sigma"]))
        assert abs(of - f) <= 1e-12 * abs(f)
        assert np.abs(og - gr).max() <= 1e-12 * np.abs(gr).max()
    for d in (2, 3):
        p = "tps%d_" % d
        cost = lo.TPSCost(g[p + "ctrl"])
        for th, f, gr in zip(g[p + "thetas"], g[p + "f"], g[p + "grad"]):
            of, og = cost(th, g[p + "ms"], g[p + "ps"], g[p + "mt"], g[p + "pt"], float(g[p + "sigma"]))
            assert abs(of - f) <= 1e-12 * abs(f)
            assert np.abs(og - gr).max() <= 1e-12 * np.abs(gr).max()


def _oracle_rigid(g, pre):
    x = lo.registration(lo.rigid_cost, np.r_[1.0, np.zeros(6)], (g[pre + "mu_s"], g[pre + "phi_s"]), (g[pre + "mu_t"], g[pre + "phi_t"]),
                        float(g[pre + "sigma"]))
    return lo.quat2mat(x[:4]), x[4:7]


def _oracle_tps(g, pre):
    cost = lo.TPSCost(g[pre + "ctrl"])
    x = lo.registration(cost, cost.initial(), (g[pre + "mu_s"], g[pre + "phi_s"]), (g[pre + "mu_t"], g[pre + "phi_t"]),
                        float(g[pre + "sigma"]))
    return cost.split(x)


def test_oracle_matches_reference_registrations():
    g = _golden()
    rot, t = _oracle_rigid(g, "bunny_")
    np.testing.assert_allclose(rot, g["bunny_rot"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(t, g["bunny_t"], rtol=0, atol=1e-8)
    a, v = _oracle_tps(g, "fish_")
    assert np.abs(a - g["fish_a"]).max() <= 1e-8 * np.abs(g["fish_a"]).max()
    assert np.abs(v - g["fish_v"]).max() <= 1e-8 * np.abs(g["fish_v"]).max()


# ---- 2. gradients against central differences -------------------------------------------------------------------------------------
def _central(fn, x, idx, h):
    out = []
    for i in idx:
        e = np.zeros_like(x)
        e[i] = h
        out.append((fn(x + e)[0] - fn(x - e)[0]) / (2.0 * h))
    return np.array(out)


def test_oracle_rigid_gradient_is_half_the_central_difference():
    """all 7 parameters.  The reference's gradient is half the derivative of f: compute_l2_dist divides by 2 sigma^2 where
    d/dmu exp(-|d|^2 / (2 sigma^2)) brings 1 / sigma^2 (cost_functions.py:40); BFGS follows that gradient, so it is kept.  At unit
    quaternions with q_2 = q_3 = 0 or q_1^2 + q_2^2 = q_0^2 + q_3^2 the reference's quaternion derivative is the exact one (see
    diff_rot_from_quaternion)."""
    g = _golden()
    args = (g["rigid_ms"], g["rigid_ps"], g["rigid_mt"], g["rigid_pt"], float(g["rigid_sigma"]))
    qs = [np.array([1.0, 0, 0, 0]), np.array([np.cos(0.3), np.sin(0.3), 0, 0]),
          np.r_[np.cos(0.4), np.cos(1.1), np.sin(1.1), np.sin(0.4)] / np.sqrt(2.0)]
    for q in qs:
        x = np.r_[q, 0.02, -0.01, 0.03]
        num = _central(lambda th: lo.rigid_cost(th, *args), x, range(7), 1e-6)
        ana = lo.rigid_cost(x, *args)[1]
        assert np.abs(0.5 * num - ana).max() <= 1e-6 * np.abs(ana).max(), (q, num, ana)


def test_reference_quaternion_derivative_departs_off_that_set():
    """a generic unit quaternion: dR_22/dq_2 and dR_22/dq_3 of the reference are not the derivative of quat2mat; every other
    entry is"""
    q = np.array([0.8, 0.1, 0.3, 0.5])
    q /= np.linalg.norm(q)
    d = se3_op.diff_rot_from_quaternion(q)
    num = np.array([(se3_op.quat2mat(q + e) - se3_op.quat2mat(q - e)) / 2e-6 for e in 1e-6 * np.identity(4)])
    bad = np.zeros((4, 3, 3), dtype=bool)
    bad[2, 2, 2] = bad[3, 2, 2] = True
    assert np.abs(num - d)[~bad].max() <= 1e-8
    assert np.abs(num - d)[bad].min() > 1e-2
    np.testing.assert_allclose(d, lo.diff_rot_from_quaternion(q), rtol=0, atol=1e-15)


@pytest.mark.parametrize("alpha,beta,factor", [(1.0, 0.0, 0.5), (0.0, 0.1, 1.0)])
def test_oracle_tps_gradient_is_central_difference(alpha, beta, factor):
    """the L2 terms' gradient is half their derivative, like the rigid one; the bending term's is its derivative"""
    g = _golden()
    for d in (2, 3):
        p = "tps%d_" % d
        cost = lo.TPSCost(g[p + "ctrl"], alpha, beta)
        args = (g[p + "ms"], g[p + "ps"], g[p + "mt"], g[p + "pt"], float(g[p + "sigma"]))
        x = g[p + "thetas"][2]
        idx = np.random.default_rng(d).choice(len(x), 12, replace=False)
        num = _central(lambda th: cost(th, *args), x, idx, 1e-6)
        ana = cost(x, *args)[1][idx]
        assert np.abs(factor * num - ana).max() <= 1e-6 * np.abs(ana).max()


def test_quat2mat_is_a_rotation():
    for q in (np.array([1.0, 0, 0, 0]), np.array([0.3, -1.2, 0.4, 2.0]), np.zeros(4)):
        r = se3_op.quat2mat(q)
        np.testing.assert_allclose(r.dot(r.T), np.identity(3), atol=1e-14)
        np.testing.assert_allclose(r, lo.quat2mat(q), atol=1e-15)
    np.testing.assert_allclose(se3_op.quat2mat(np.r_[np.cos(0.25), 0, 0, np.sin(0.25)]), _rot([0, 0, 1], np.rad2deg(0.5)), atol=1e-15)


# ---- 3. cpd_gmm_fit against the oracle --------------------------------------------------------------------------------------------
def _check_fit(x, k, seed=0, seeds=None, max_iter=100, twice=True):
    seeds = lo.random_from_data(len(x), k, seed) if seeds is None else np.asarray(seeds)
    h = _cabi.Handle(x.shape[1])
    h.set_source(x)
    w, mu, var, it, lb = h.gmm_fit(k, seeds, max_iter=max_iter)
    ow, omu, ovar, oit, olb = lo.gmm_fit(x, k, seeds=seeds, max_iter=max_iter)
    assert it == oit
    worst = 0.0
    for a, b in ((w, ow), (mu, omu), (var, ovar)):
        err = np.abs(a - b).max() / np.abs(b).max()
        worst = max(worst, err)
        assert err <= REL, err
    np.testing.assert_allclose(lb, olb, rtol=REL, atol=0)
    if twice:
        again = h.gmm_fit(k, seeds, max_iter=max_iter)
        for a, b in zip((w, mu, var, it, lb), again):
            np.testing.assert_array_equal(a, b)
    print("gmm fit n=%d k=%d iterations %d worst relative error %.3g" % (len(x), k, it, worst))
    return w, mu, var, it, lb


def _dup_cloud():
    x = _lumps(600, 3, 11)
    x = np.vstack([x, x[:40]])             # duplicates: seeds 600.. coincide with 0..
    seeds = np.r_[np.arange(0, 20), np.arange(600, 620), np.arange(100, 140)]
    return x, seeds


def _outlier_cloud():
    x = _lumps(400, 3, 12)
    x[17] = [6.0, -5.0, 4.0]               # a far outlier (tens of widths away), one of the seeds
    return x


def test_gmm_fit_bunny_emulated(emulated):
    _check_fit(_bunny(), 60, 1)


def test_gmm_fit_lumps_emulated(emulated):
    _check_fit(_lumps(900, 3, 2), 40, 2)


def test_gmm_fit_2d_emulated(emulated):
    _check_fit(_lumps(700, 2, 3), 30, 3)


def test_gmm_fit_duplicate_seeds_emulated(emulated):
    x, seeds = _dup_cloud()
    _check_fit(x, len(seeds), seeds=seeds)


def test_gmm_fit_edges_emulated(emulated):
    x = _lumps(300, 3, 4)
    _check_fit(x, 1, 0)
    _check_fit(x[:120], 120, 0, max_iter=8)            # K = N
    _check_fit(_outlier_cloud(), 25, seeds=np.r_[17, np.arange(30, 54)])


# ---- 4. cpd_l2_dist against the oracle --------------------------------------------------------------------------------------------
def _check_l2(ns, nt, dim, seed, sigma=0.2, far=False, same=False):
    rng = np.random.default_rng(seed)
    ms = rng.standard_normal((ns, dim)) * 0.5
    mt = ms if same else rng.standard_normal((nt, dim)) * 0.5 + 0.1
    ps = rng.dirichlet(np.ones(ns))
    pt = ps if same else rng.dirichlet(np.ones(len(mt)))
    if far:
        mt = mt.copy()
        mt[: len(mt) // 3] += 40.0             # these pairs underflow to exactly 0
    f, g = _cabi.l2_dist(ms, ps, mt, pt, sigma)
    of, og = lo.l2_dist(ms, ps, mt, pt, sigma)
    assert abs(f - of) <= 1e-12 * abs(of)
    assert np.abs(g - og).max() <= 1e-11 * np.abs(og).max()
    f2, g2 = cost_functions.compute_l2_dist(ms, ps, mt, pt, sigma)
    assert f2 == f and np.array_equal(g2, g)


@pytest.mark.parametrize("ns,nt,dim,far,same", [(800, 800, 3, False, False), (193, 257, 3, False, False), (131, 67, 2, False, False),
                                                (300, 300, 3, False, True), (150, 120, 3, True, False)])
def test_l2_dist_matches_oracle_emulated(emulated, ns, nt, dim, far, same):
    _check_l2(ns, nt, dim, ns + nt, far=far, same=same)


# ---- 5. cpd_tps_kernel ------------------------------------------------------------------------------------------------------------
def _check_tps():
    rng = np.random.default_rng(8)
    for d in (2, 3):
        x = rng.standard_normal((57, d))
        y = np.vstack([x[:7], x[7:10] + 1e-5, rng.standard_normal((70, d))])     # r^2 = 0 and r^2 <= 1e-9 for 2-D
        got = math_utils.tps_kernel(x, y)
        assert got.dtype == np.float32
        np.testing.assert_array_equal(got, lo.tps_kernel(x, y))
    with pytest.raises(ValueError):
        math_utils.tps_kernel(np.zeros((3, 4)), np.zeros((3, 4)))


def test_tps_kernel_bit_identical_emulated(emulated):
    _check_tps()


# ---- 6. the registrations with the reference's features replayed ------------------------------------------------------------------
class _Replay(features.Feature):
    """hands out the given (means, weights) in order"""

    def __init__(self, feats):
        self._feats, self._k = list(feats), 0

    def init(self):
        pass

    def compute(self, data):
        out = self._feats[self._k % len(self._feats)]
        self._k += 1
        return out


def _check_replay():
    g = _golden()
    bunny = _bunny()
    reg = l2dist_regs.L2DistRegistration(bunny, _Replay([(g["bunny_mu_s"], g["bunny_phi_s"]), (g["bunny_mu_t"], g["bunny_phi_t"])]),
                                         cost_functions.RigidCostFunction())
    assert abs(reg._sigma - float(g["bunny_sigma"])) <= 1e-14 * float(g["bunny_sigma"])
    res = reg.registration(g["bunny_target"])
    np.testing.assert_allclose(res.rot, g["bunny_rot"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(res.t, g["bunny_t"], rtol=0, atol=1e-6)
    fish_s = np.loadtxt(_golden_path("data/fish_source.txt"))
    cost = cost_functions.TPSCostFunction(g["fish_ctrl"])
    reg = l2dist_regs.L2DistRegistration(fish_s, _Replay([(g["fish_mu_s"], g["fish_phi_s"]), (g["fish_mu_t"], g["fish_phi_t"])]), cost)
    res = reg.registration(np.loadtxt(_golden_path("data/fish_target.txt")))
    for a, b in ((res.a, g["fish_a"]), (res.v, g["fish_v"])):
        assert np.abs(a - b).max() <= 1e-6 * np.abs(b).max()


def _golden_path(name):
    import os

    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name)


def _check_against_oracle_loop():
    """device features on the same seed, then the package's loop against the oracle's on those features"""
    bunny = _bunny()
    tgt = bunny.dot(_rot([0.0, 1.0, 1.0], 15.0).T) + [0.01, 0.0, -0.01]
    reg = l2dist_regs.RigidGMMReg(bunny, n_gmm_components=120, seed=4)
    seen = []
    reg._feature_gen = _Recorder(reg._feature_gen, seen)
    res = reg.registration(tgt)
    (ms, ps), (mt, pt) = seen
    sigma = lo.estimate_sigma(bunny)
    x = lo.registration(lo.rigid_cost, np.r_[1.0, np.zeros(6)], (ms, ps), (mt, pt), sigma)
    np.testing.assert_allclose(res.rot, lo.quat2mat(x[:4]), rtol=0, atol=1e-6)
    np.testing.assert_allclose(res.t, x[4:7], rtol=0, atol=1e-6)


class _Recorder(features.Feature):
    def __init__(self, inner, seen):
        self._inner, self._seen = inner, seen

    def init(self):
        self._inner.init()

    def compute(self, data):
        out = self._inner.compute(data)
        self._seen.append(out)
        return out


def test_registration_replay_matches_reference_emulated(emulated):
    _check_replay()


def test_registration_matches_oracle_loop_emulated(emulated):
    _check_against_oracle_loop()


# ---- 7. known answer ---------------------------------------------------------------------------------------------------------------
KNOWN_ROT, KNOWN_T = _rot([1.0, -0.5, 2.0], 30.0), np.array([0.02, -0.015, 0.01])


def _angle(a, b):
    return np.rad2deg(np.arccos(np.clip((np.trace(a.T.dot(b)) - 1.0) / 2.0, -1.0, 1.0)))


def _check_known(res, src):
    extent = np.ptp(src, axis=0).max()
    assert _angle(res.rot, KNOWN_ROT) <= 1.0, _angle(res.rot, KNOWN_ROT)
    assert np.abs(res.t - KNOWN_T).max() <= 1e-2 * extent


def _oracle_known(maxiter):
    src = _bunny()
    tgt = src.dot(KNOWN_ROT.T) + KNOWN_T
    k = int(len(src) * 0.8)
    ws, ms = lo.gmm_fit(src, k, 0)[:2]
    wt, mt = lo.gmm_fit(tgt, k, 0)[:2]
    x = lo.registration(lo.rigid_cost, np.r_[1.0, np.zeros(6)], (ms, ws), (mt, wt), lo.estimate_sigma(src), maxiter=maxiter)
    return transformation.RigidTransformation(lo.quat2mat(x[:4]), x[4:7])


def test_known_answer_oracle():
    """the reference's single outer iteration stops about 4.6 degrees short of 30; ten outer iterations (sigma annealed by 0.9
    each) recover the motion"""
    _check_known(_oracle_known(10), _bunny())
    assert _angle(_oracle_known(1).rot, KNOWN_ROT) > 1.0


def _check_known_device():
    src = _bunny()
    tgt = src.dot(KNOWN_ROT.T) + KNOWN_T
    res = l2dist_regs.RigidGMMReg(src).registration(tgt, maxiter=10)
    _check_known(res, src)
    np.testing.assert_allclose(res.rot, _oracle_known(10).rot, rtol=0, atol=1e-6)
    seen = []
    res = l2dist_regs.registration_gmmreg(src, tgt, callbacks=[seen.append])     # the reference's defaults: one outer iteration
    assert len(seen) >= 1 and isinstance(seen[-1], transformation.RigidTransformation)
    np.testing.assert_allclose(res.rot, _oracle_known(1).rot, rtol=0, atol=1e-6)
    np.testing.assert_allclose(res.t, _oracle_known(1).t, rtol=0, atol=1e-6)


def test_known_answer_emulated(emulated):
    _check_known_device()


# ---- 8. refusals and the Python surface -------------------------------------------------------------------------------------------
def _check_refusals():
    x = _lumps(200, 3, 9)
    h = _cabi.Handle(3)
    with pytest.raises(_cabi.CpdError, match="source"):
        h.gmm_fit(3, [0, 1, 2])
    h.set_source(x)
    for k in (0, 201):
        with pytest.raises(_cabi.CpdError, match="n_components"):
            h.gmm_fit(k, np.arange(k) % 200)
    for bad in ([0, 1, 1], [0, -1, 2], [0, 1, 200]):
        with pytest.raises(_cabi.CpdError, match="seed"):
            h.gmm_fit(3, bad)
    with pytest.raises(_cabi.CpdError, match="reg_covar"):
        h.gmm_fit(3, [0, 1, 2], reg_covar=-1e-6)
    with pytest.raises(_cabi.CpdError, match="max_iter"):
        _cabi.check(h._lib.cpd_gmm_fit(h._h, 3, np.arange(3, dtype=np.int64).ctypes.data_as(_cabi.ctypes.POINTER(_cabi.ctypes.c_int64)),
                                       1e-6, 1e-3, 0, None, None, None, None, None))
    xb = x.copy()
    xb[5, 2] = np.nan
    hb = _cabi.Handle(3)
    hb.set_source(xb)
    with pytest.raises(_cabi.CpdError, match="non-finite"):
        hb.gmm_fit(3, [0, 1, 2])
    ms, ps = x[:10], np.full(10, 0.1)
    for args, pat in (((ms, ps, ms, ps, 0.0), "sigma"), ((ms, ps, ms, ps, np.inf), "sigma"),
                      ((ms[:, :1], ps, ms[:, :1], ps, 0.1), "dim"), ((np.r_[ms[:9], [[np.nan] * 3]], ps, ms, ps, 0.1), "non-finite")):
        with pytest.raises(_cabi.CpdError, match=pat):
            _cabi.l2_dist(*args)
    with pytest.raises(ValueError):
        _cabi.l2_dist(ms, ps[:5], ms, ps, 0.1)
    with pytest.raises(_cabi.CpdError, match="TPS"):
        _cabi.check(_cabi.lib().cpd_tps_kernel(0, _cabi.dptr(ms), 10, _cabi.dptr(ms), 10, 4, None))


def _check_surface():
    src = _lumps(300, 3, 10)
    tgt = src.dot(_rot([0, 0, 1], 8.0).T)
    with pytest.raises(ValueError, match="Unknown transform type"):
        l2dist_regs.registration_gmmreg(src, tgt, tf_type_name="affine")
    gm = features.GMM(40, seed=3)
    mu, w = gm(src)
    assert mu.shape == (40, 3) and w.shape == (40,) and abs(w.sum() - 1.0) <= 1e-12
    np.testing.assert_array_equal(gm.seeds(300), np.random.RandomState(3).choice(300, 40, replace=False))
    assert gm.n_iter_ == len(gm.lower_bounds_) and gm.covariances_.shape == (40,)
    reg = l2dist_regs.RigidGMMReg(src, n_gmm_components=800)
    assert reg._feature_gen._n_gmm_components == 240                # min(800, 0.8 N)
    seen = []
    reg.set_callbacks([seen.append])
    res = reg.registration(tgt)
    assert len(seen) >= 2 and isinstance(res, transformation.RigidTransformation)
    src2 = _lumps(120, 2, 13)
    tps = l2dist_regs.TPSGMMReg(src2, n_gmm_components=30)
    np.testing.assert_array_equal(tps._cost_fn._control_pts, tps._source_features()[0])
    seen = []
    res = l2dist_regs.registration_gmmreg(src2, src2 * 1.05, tf_type_name="nonrigid", callbacks=[seen.append], n_gmm_components=30)
    assert isinstance(res, transformation.TPSTransformation) and res.a.shape == (3, 2) and res.v.shape == (27, 2) and seen
    moved = res.transform(src2)
    assert moved.shape == src2.shape and np.isfinite(moved).all()
    for name in ("L2DistRegistration", "RigidGMMReg", "TPSGMMReg", "registration_gmmreg"):
        assert hasattr(l2dist_regs, name)
    for name in ("CostFunction", "compute_l2_dist", "RigidCostFunction", "TPSCostFunction"):
        assert hasattr(cost_functions, name)


def test_refusals_emulated(emulated):
    _check_refusals()


def test_python_surface_emulated(emulated):
    _check_surface()


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_small_cases_gpu(bunny):
    _check_fit(_bunny(), 60, 1)
    _check_fit(_lumps(900, 3, 2), 40, 2)
    _check_fit(_lumps(700, 2, 3), 30, 3)
    x, seeds = _dup_cloud()
    _check_fit(x, len(seeds), seeds=seeds)
    x = _lumps(300, 3, 4)
    _check_fit(x, 1, 0)
    _check_fit(x[:120], 120, 0, max_iter=8)
    _check_fit(_outlier_cloud(), 25, seeds=np.r_[17, np.arange(30, 54)])
    for ns, nt, dim, far, same in [(800, 800, 3, False, False), (193, 257, 3, False, False), (131, 67, 2, False, False),
                                   (300, 300, 3, False, True), (150, 120, 3, True, False)]:
        _check_l2(ns, nt, dim, ns + nt, far=far, same=same)
    _check_tps()
    _check_refusals()
    _check_surface()


@pytest.mark.gpu
def test_registrations_gpu():
    _check_replay()
    _check_against_oracle_loop()
    _check_known_device()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_gmm_fit_100k_gpu():
    _check_fit(_lumps(100_000, 3, 20), 800, 5, max_iter=5, twice=False)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_gmm_fit_1m_gpu():
    import torch

    x = _lumps(1_000_000, 3, 21)
    seeds = lo.random_from_data(len(x), 800, 6)
    out = []
    for _ in range(2):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        h = _cabi.Handle(3)
        h.set_source(x)
        out.append(h.gmm_fit(800, seeds))
        used = free0 - torch.cuda.mem_get_info(0)[0]
        h.close()
    w, mu, var, it, lb = out[0]
    for a, b in zip(out[0], out[1]):
        np.testing.assert_array_equal(a, b)
    assert abs(w.sum() - 1.0) <= 1e-12
    assert (var >= 1e-6).all()
    assert (np.diff(lb) >= -1e-12 * np.abs(lb[1:])).all()
    print("1M points, K = 800: %d iterations, lower bound %.9g, device memory of the handle and fit after it %.1f MB"
          % (it, lb[-1], used / 2 ** 20))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_l2_dist_10k_gpu():
    _check_l2(10_000, 12_000, 3, 77, sigma=0.1)
