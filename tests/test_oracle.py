"""The oracle (oracle/cpd_oracle.py) against fixtures produced by the reference itself
(tests/golden/make_golden.py).  CPU only."""
import numpy as np
import pytest

from oracle import cpd_oracle as orc
from conftest import load_golden


def test_known_answer_squared_kernel_sum():
    # reference tests/test_math_utils.py:6-11
    g = load_golden("math_utils.npz")
    x = g["x"]
    brute = np.sum([np.sum((x[i] - x) ** 2) for i in range(5)]) / (5 * 5 * 3)
    assert orc.sigma2_init(x, x) == pytest.approx(brute, abs=1e-7)
    assert orc.sigma2_init(x, x) == float(g["sks"])
    assert orc.sigma2_init_exact(x, x) == pytest.approx(brute, rel=1e-14)


def test_rbf_symmetric_and_golden():
    # reference tests/test_math_utils.py:13-16
    g = load_golden("math_utils.npz")
    k = orc.rbf_kernel_f32(g["x"] * 0.1, g["x"] * 0.1, 1.0)
    assert np.allclose(k, k.T)
    assert np.array_equal(k, g["rbf"])


def test_init_matches_reference(bunny):
    s2 = orc.sigma2_init(bunny["source"], bunny["target"])
    assert s2 == float(bunny["init_sigma2"])            # float32 value, bit-exact
    assert s2 == pytest.approx(0.0036908406764268875, rel=1e-12)   # the reference's value
    assert orc.sigma2_init_exact(bunny["source"], bunny["target"]) == pytest.approx(s2, rel=2e-7)
    q0 = 1.0 + bunny["target"].shape[0] * 3 * 0.5 * np.log(np.float32(s2))
    assert float(q0) == pytest.approx(float(bunny["init_q"]), rel=1e-12)


@pytest.mark.parametrize("tag,w", [("e0", 0.0), ("e0w", 0.3)])
def test_estep_matches_reference(bunny, tag, w):
    es = orc.expectation_step(bunny["source"], bunny["target"], float(bunny["init_sigma2"]), w)
    assert np.array_equal(es.pt1, bunny[tag + "_pt1"])
    np.testing.assert_allclose(es.p1, bunny[tag + "_p1"], rtol=1e-14)
    np.testing.assert_allclose(es.px, bunny[tag + "_px"], rtol=1e-13, atol=1e-16)
    assert es.n_p == pytest.approx(float(bunny[tag + "_np"]), rel=1e-14)


def test_estep_blocking_is_exact(syn1500):
    ts, tgt = syn1500["es_tsource"], syn1500["target_outl"]
    for tag in ("dead", "deadw", "mid"):
        s2, w = float(syn1500["es_%s_sigma2" % tag]), float(syn1500["es_%s_w" % tag])
        for block in (None, 77):
            es = orc.expectation_step(ts, tgt, s2, w, block=block)
            np.testing.assert_allclose(es.pt1, syn1500["es_%s_pt1" % tag], rtol=1e-14, atol=0)
            np.testing.assert_allclose(es.p1, syn1500["es_%s_p1" % tag], rtol=1e-12, atol=1e-300)
            np.testing.assert_allclose(es.px, syn1500["es_%s_px" % tag], rtol=1e-12, atol=1e-300)
    # the dead-column case really has dead columns (reference semantics cpd.py:81)
    assert float(syn1500["es_dead_np"]) < tgt.shape[0] - 1


def test_shard_uses_global_n(syn1500):
    ts, tgt = syn1500["es_tsource"], syn1500["target_outl"]
    full = orc.expectation_step(ts, tgt, 3e-3, 0.2)
    h = tgt.shape[0] // 2
    a = orc.expectation_step(ts, tgt[:h], 3e-3, 0.2, n_global=tgt.shape[0])
    b = orc.expectation_step(ts, tgt[h:], 3e-3, 0.2, n_global=tgt.shape[0])
    np.testing.assert_allclose(a.p1 + b.p1, full.p1, rtol=1e-12)
    np.testing.assert_allclose(np.r_[a.pt1, b.pt1], full.pt1, rtol=1e-15)


CASES = [
    ("bunny.npz", "rigid10", "rigid", 10, 0.0, {}, "source", "target"),
    ("bunny.npz", "rigid10_w01", "rigid", 10, 0.1, {}, "source", "target"),
    ("bunny.npz", "rigid10_noscale", "rigid", 10, 0.0, {"update_scale": False}, "source", "target"),
    ("bunny.npz", "affine10", "affine", 10, 0.0, {}, "source", "target"),
    ("synthetic1500.npz", "rigid20", "rigid", 20, 0.0, {}, "source", "target"),
    ("synthetic1500.npz", "rigid20_outl_w", "rigid", 20, 0.2, {}, "source", "target_outl"),
    ("synthetic1500.npz", "rigid30_outl_w0", "rigid", 30, 0.0, {}, "source", "target_outl"),
    ("synthetic1500.npz", "affine20", "affine", 20, 0.0, {}, "source_a", "target_a"),
    ("nonrigid.npz", "fish15", "nonrigid", 15, 0.0, {"beta": 2.0, "lmd": 2.0}, "fish_source", "fish_target"),
    ("nonrigid.npz", "fishaffine15", "affine", 15, 0.0, {}, "fish_source", "fish_target"),
    ("nonrigid.npz", "fishrigid15", "rigid", 15, 0.0, {}, "fish_source", "fish_target"),
    ("nonrigid.npz", "nr12", "nonrigid", 12, 0.0, {"beta": 0.5, "lmd": 1.0}, "nr_source", "nr_target"),
    ("nonrigid.npz", "nrc8", "nonrigid_constrained", 8, 0.0, {"beta": 0.5, "lmd": 1.0, "alpha": 1e-2}, "nr_source", "nr_target"),
]


@pytest.mark.parametrize("fname,tag,tf_type,iters,w,kw,sk,tk", CASES)
def test_fixed_iteration_registration(fname, tag, tf_type, iters, w, kw, sk, tk):
    g = load_golden(fname)
    kw = dict(kw)
    if tf_type == "nonrigid_constrained":
        kw["idx_source"], kw["idx_target"] = g["nrc_idx_source"], g["nrc_idx_target"]
    res, it = orc.registration(g[sk], g[tk], tf_type, w=w, maxiter=iters, tol=-1.0, **kw)
    assert it == iters
    assert res.sigma2 == pytest.approx(float(g[tag + "_sigma2"]), rel=1e-9)
    assert res.q == pytest.approx(float(g[tag + "_q"]), rel=1e-9)
    if tf_type == "rigid":
        np.testing.assert_allclose(res.params[0], g[tag + "_rot"], atol=1e-10)
        np.testing.assert_allclose(res.params[1], g[tag + "_t"], atol=1e-10)
        assert res.params[2] == pytest.approx(float(g[tag + "_scale"]), rel=1e-10)
    elif tf_type == "affine":
        np.testing.assert_allclose(res.params[0], g[tag + "_b"], atol=1e-9)
        np.testing.assert_allclose(res.params[1], g[tag + "_t"], atol=1e-9)
    else:
        np.testing.assert_allclose(res.params[0], g[tag + "_w"], rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("tag,tf_type", [("rigid_default", "rigid"), ("affine_default", "affine")])
def test_default_tolerance_iteration_count(bunny, tag, tf_type):
    res, it = orc.registration(bunny["source"], bunny["target"], tf_type)
    assert it == int(bunny[tag + "_iters"])
    assert res.sigma2 == pytest.approx(float(bunny[tag + "_sigma2"]), rel=1e-9)
    # noise-free data ends on the eps32 floor of sigma2, where q is a tiny residual
    # divided by 2.4e-7: conditioned to ~1e-7 only
    assert res.q == pytest.approx(float(bunny[tag + "_q"]), rel=1e-6)


def test_appendix_c_values(bunny):
    # values regenerated by the reference itself (tests/golden/make_golden.py)
    assert int(bunny["rigid_default_iters"]) == 18
    assert float(bunny["rigid_default_sigma2"]) == pytest.approx(1.1920928955078125e-07)
    assert float(bunny["rigid10_sigma2"]) == pytest.approx(3.9235098811641994e-05, rel=1e-9)
    assert float(bunny["rigid10_scale"]) == pytest.approx(0.9571492390382025, rel=1e-10)


def test_c_oracle_matches_numpy_oracle(syn1500):
    from oracle import c_oracle
    ts, tgt = syn1500["es_tsource"], syn1500["target_outl"]
    for s2, w in [(1e-4, 0.0), (1e-4, 0.1), (3e-3, 0.0), (0.2, 0.3)]:
        a = orc.expectation_step(ts, tgt, s2, w)
        b = c_oracle.expectation_step(ts, tgt, s2, w)
        np.testing.assert_allclose(b.pt1, a.pt1, rtol=1e-11, atol=0)   # libm exp vs numpy SIMD exp
        np.testing.assert_allclose(b.p1, a.p1, rtol=1e-11, atol=1e-300)
        np.testing.assert_allclose(b.px, a.px, rtol=1e-11, atol=1e-300)
        assert b.n_p == pytest.approx(a.n_p, rel=1e-13)
    fs = np.random.default_rng(0).random((50, 2))
    a = orc.expectation_step(fs, fs[::-1] + 0.01, 0.02, 0.1)
    b = c_oracle.expectation_step(fs, fs[::-1] + 0.01, 0.02, 0.1)
    np.testing.assert_allclose(b.p1, a.p1, rtol=1e-12)


def test_bench_workload_is_the_oracles():
    from probreg_b200 import synthetic
    for kind in ("rigid", "affine"):
        a = orc.synthetic_pair(777, kind)
        b = synthetic.synthetic_pair(777, kind)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_constrained_prior_terms_follow_numpy_indexing():
    """ConstrainedNonRigidCPD builds p1_tilde / px_tilde of cpd.py:364-374 as a sparse gather; the reference's dense
    `p_tilde[idx_source, idx_target] = 1` accepts anything NumPy advanced indexing accepts (broadcasting, negative indices,
    boolean masks) -- the gather must give the same two sums.  Host-only: no device call is made by _prior_terms."""
    from probreg_b200 import cpd

    rng = np.random.default_rng(5)
    m, n = 17, 23
    src, tgt = rng.random((m, 3)), rng.random((n, 3))
    mask = np.zeros(m, dtype=bool)
    mask[[2, 5, 11]] = True
    cases = [
        (np.array([0, 3, 3, 9]), np.array([1, 4, 4, 20])),              # equal length, a duplicate pair
        (np.array([0, 3, 9]), 7),                                        # scalar broadcasts
        (np.array([-1, -17, 4]), np.array([-23, 5, -1])),                # negative indices
        (mask, np.array([6, 7, 8])),                                     # boolean mask on the source axis
        (np.array([[0], [1]]), np.array([[2, 3, 4]])),                   # 2-D broadcast: 2 x 3 pairs
    ]
    for isrc, itgt in cases:
        obj = cpd.ConstrainedNonRigidCPD.__new__(cpd.ConstrainedNonRigidCPD)
        obj._source, obj.idx_source, obj.idx_target = src, isrc, itgt
        obj._prior_terms(tgt)
        dense = np.zeros((m, n))
        dense[isrc, itgt] = 1.0
        np.testing.assert_allclose(obj.p1_tilde, dense.sum(axis=1))
        np.testing.assert_allclose(obj.px_tilde, dense.dot(tgt), atol=1e-15)
    obj.idx_source, obj.idx_target = np.array([0.5]), np.array([1])
    with pytest.raises(IndexError):
        obj._prior_terms(tgt)
    obj.idx_source, obj.idx_target = np.array([m]), np.array([1])
    with pytest.raises(IndexError):
        obj._prior_terms(tgt)
