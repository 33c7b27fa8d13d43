"""FilterReg: the permutohedral lattice, the E-step and the registration loop against oracle/filterreg_oracle.py.

The lattice is held to bit identity: the device against the reference's own lattice (oracle/_ref, built from the unmodified
permutohedral.cpp) and against the oracle's numpy float32 restatement, which is itself held to oracle/_ref.  CPU cases run the device
code under the emulation (tests/emu); the gpu-marked cases run it on the H100 at full size.
"""
import numpy as np
import pytest

from oracle import filterreg_oracle as fo
from probreg_b200 import _cabi, filterreg, gaussian_filtering

needs_ref = pytest.mark.skipif(not fo.ref_available(), reason="oracle/_ref was not built (build() with $PROBREG_REFERENCE)")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _same(a, b):
    return a is None and b is None or np.array_equal(_bits(a), _bits(b))


def _lattice_cases():
    """(name, feature, values, with_blur): the edges of the lattice."""
    rng = np.random.default_rng(3)
    out = []
    for d in (2, 3):
        for n in (8, 9, 10, 11):                              # (M+N) % 4 = 0..3, near the origin: the padding vertices matter
            f = rng.standard_normal((n, d)) * 0.6
            for vs in (1, 2, 3, 4):
                for blur in (True, False):
                    out.append(("origin-d%d-n%d-vs%d-%s" % (d, n, vs, blur), f, rng.standard_normal((n, vs)), blur))
        far = rng.standard_normal((37, d)) * 300.0 + 40000.0   # elevated keys beyond 32767 wrap to 16 bits
        out.append(("wrap-d%d" % d, far, rng.standard_normal((37, 3)), True))
        dup = np.repeat(rng.standard_normal((6, d)), 3, axis=0)
        out.append(("duplicates-d%d" % d, dup, rng.standard_normal((18, 2)), True))
        out.append(("single-d%d" % d, rng.standard_normal((1, d)), np.ones((1, 1)), True))
    f = np.array([[100.0, 50.0, 30.0]] * 5) + rng.standard_normal((5, 3)) * 0.01   # 5 points: a lattice of 8, 4 points: 4
    out.append(("phantom-5", f, np.ones((5, 1)), True))
    out.append(("phantom-4", f[:4], np.ones((4, 1)), True))
    return out


CASES = _lattice_cases()


@needs_ref
def test_numpy_lattice_is_the_reference_bit_for_bit():
    for name, f, v, blur in CASES:
        a, sa = fo.ref_filter(f, v, blur)
        b, sb = fo.lattice_filter(f, v, blur)
        assert sa == sb, name
        assert _same(a, b), name
    f = CASES[-2][1]
    assert fo.ref_lattice_size(f) == 8 and fo.ref_lattice_size(f[:4]) == 4


def test_dropped_padding_lane_changes_the_result_and_the_tie_rule_does_not():
    """A dropped padding lane fails at least one case.  The tie rule of the rounding cannot: a remainder-0 point rounded the other
    way at a tie changes the coordinate sum by one, and the rank correction (permutohedral.cpp:237-243) moves it back, so the
    simplex, its keys and its weights come out the same.  Shown on the cases and on an exact tie."""
    def differs(**kw):
        for name, f, v, blur in CASES:
            a, sa = fo.lattice_filter(f, v, blur)
            b, sb = fo.lattice_filter(f, v, blur, **kw)
            if sa != sb or not _same(a, b):
                return True
        # an exact tie of the rounding: a 2-D point whose first elevated coordinate / 3 is 1.5 in float32
        f32 = np.float32
        sf0 = f32(1.0 / np.sqrt(2.0) * float(f32(np.sqrt(2.0 / 3.0) * 3)))
        x = f32(4.5) / sf0
        for _ in range(64):
            if f32(1.0) / f32(3) * (x * sf0) == f32(1.5):
                break
            x = np.nextafter(x, f32(np.inf), dtype=f32)
        assert f32(1.0) / f32(3) * (x * sf0) == f32(1.5)
        f = np.array([[x, 0.0], [0.1, 0.2], [-0.3, 0.1], [0.2, -0.2]])
        a, sa = fo.lattice_filter(f, np.ones((4, 1)))
        b, sb = fo.lattice_filter(f, np.ones((4, 1)), **kw)
        return sa != sb or not _same(a, b)

    assert differs(pad_lane=False)
    assert not differs(rounding="ties_down")


def _check_device_lattice():
    for name, f, v, blur in CASES:
        ref, sr = fo.ref_filter(f, v, blur) if fo.ref_available() else fo.lattice_filter(f, v, blur)
        out, size = _cabi.lattice_filter(f, v, blur)
        assert size == sr, name
        assert _same(out, ref), name
        ph = gaussian_filtering.Permutohedral(f, blur)
        assert ph.get_lattice_size() == sr and _same(ph.filter(v, 3), ref), name


def test_device_lattice_bit_identical_emulated(emulated):
    _check_device_lattice()


def _clouds(m, n, d, seed=0, spread=0.3):
    rng = np.random.default_rng(seed)
    src = rng.standard_normal((m, d)) * spread
    th = 0.3
    r = np.identity(d)
    r[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
    tgt = (rng.standard_normal((n, d)) * spread).dot(r.T) + 0.05
    nrm = rng.standard_normal((n, d))
    return src, tgt, nrm / np.linalg.norm(nrm, axis=1)[:, None]


def _impl():
    return "ref" if fo.ref_available() else "numpy"


def _check_estep(src, tgt, nrm, sigma2, expect_blur=None):
    for upd in (False, True):
        for normals in (None, nrm):
            a = _cabi.filterreg_estep(src, tgt, sigma2, upd, normals)
            b = fo.expectation_step(src, tgt, sigma2, upd, normals, impl=_impl())
            assert a[4] == b[4]
            if expect_blur is not None:
                assert a[4] == expect_blur
            for x, y in zip(a[:4], b[:4]):
                assert _same(x, y)


def test_estep_bit_identical_emulated(emulated):
    src, tgt, nrm = _clouds(61, 1000, 3)
    _check_estep(src, tgt, nrm, 50.0, True)             # few vertices (<= n * alpha = 15): blurred
    _check_estep(src, tgt, nrm, 0.05, False)            # more vertices: rebuilt without blur
    s2, t2, n2 = _clouds(33, 700, 2, seed=1)
    _check_estep(s2, t2, n2, 50.0, True)
    _check_estep(s2, t2, n2, 1e-4, False)
    # the public method, with the reference's argument order
    es = filterreg.RigidFilterReg(src, nrm).expectation_step(src, tgt, tgt, 50.0, True, "pt2pl")
    b = fo.expectation_step(src, tgt, 50.0, True, nrm, impl=_impl())
    assert all(_same(x, y) for x, y in zip(es, b[:4]))
    assert es.m0.dtype == np.float32 and es.m1.shape == (61, 3)


def _loop(src, tgt, nrm, objective, upd, w, sigma2, init, maxiter=20, tol=-1.0):
    """The device loop (the public class) and the oracle loop; the device loop's E-step is compared with the oracle's, bit for
    bit, at every iteration (the callback reads it from the device)."""
    params = {} if init is None else {"rot": init[0], "t": init[1]}
    calls, esteps = [], []
    reg = filterreg.RigidFilterReg(src, nrm, sigma2, upd, tf_init_params=params)
    reg.set_callbacks([lambda tfp: (calls.append(tfp), esteps.append(reg._loop.last_estep()))])
    res = reg.registration(tgt, w=w, objective_type=objective, maxiter=maxiter, tol=tol)
    s2 = sigma2 if sigma2 is not None else max(filterreg.mu.squared_kernel_sum(src, tgt), 1e-4)   # the same start on both sides
    trace = []
    rot, t, s2o, q, it = fo.registration(src, tgt, nrm, s2, upd, w, objective, maxiter, tol, 1e-4,
                                         None if init is None else init[0], None if init is None else init[1], impl=_impl(),
                                         trace=trace)
    for a, b in zip(esteps, trace):
        assert a[4] == b[4]
        assert all(_same(x, y) for x, y in zip(a[:4], b[:4] if objective == "pt2pl" else (b[0], b[1], b[2], None)))
    return res, calls, (rot, t, s2o, q, it)


def _check_loops():
    src, tgt, nrm = _clouds(90, 80, 3, seed=4)
    s2d, t2d, _ = _clouds(60, 50, 2, seed=5)
    th = 0.1
    init = (np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1.0]]), np.array([0.01, 0.0, -0.02]))
    cases = [("pt2pt", src, tgt, None, None), ("pt2pl", src, tgt, nrm, None), ("pt2pt", s2d, t2d, None, None),
             ("pt2pt", src, tgt, None, init), ("pt2pl", src, tgt, nrm, init)]
    for objective, s, t, n, ini in cases:
        for upd in (False, True):
            for w in (0.0, 0.1):
                for sigma2 in (None, 0.05):
                    res, calls, (rot, tt, s2, q, it) = _loop(s, t, n, objective, upd, w, sigma2, ini)
                    assert len(calls) == it == 20
                    np.testing.assert_allclose(res.transformation.rot, rot, rtol=0, atol=1e-9)
                    np.testing.assert_allclose(res.transformation.t, tt, rtol=0, atol=1e-9)
                    assert abs(res.sigma2 - s2) <= 1e-9 * abs(s2)
                    assert abs(res.q - q) <= 1e-9 * abs(q) + 1e-12


def test_loop_matches_oracle_emulated(emulated):
    _check_loops()


def test_loop_edges_emulated(emulated):
    _check_loop_edges()


def _check_loop_edges():
    src, tgt, nrm = _clouds(40, 44, 3, seed=6)
    # the tol stop at the oracle's iteration
    res, calls, (rot, t, s2, q, it) = _loop(src, tgt, None, "pt2pt", True, 0.0, None, None, maxiter=50, tol=5.0)
    assert len(calls) == it and it < 50
    np.testing.assert_allclose(res.transformation.rot, rot, atol=1e-9)
    # a source far from every target has m0 == 0 and is dropped
    far = np.r_[src, [[50.0, 50.0, 50.0]]]
    es = filterreg.RigidFilterReg(far).expectation_step(far, tgt, tgt, 1e-3, False)
    assert es.m0[-1] == 0
    res, _, (rot, t, _, _, _) = _loop(far, tgt, None, "pt2pt", False, 0.0, 0.01, None, maxiter=3)
    np.testing.assert_allclose(res.transformation.rot, rot, atol=1e-9)
    # every m0 zero: the loop stops at once with the previous q (None) and the initial transformation
    res = filterreg.registration_filterreg(src + 100.0, tgt, sigma2=1e-4, maxiter=5)
    assert res.q is None and np.array_equal(res.transformation.rot, np.identity(3))


def test_refusals_and_reference_errors_emulated(emulated):
    src, tgt, nrm = _clouds(10, 10, 3)
    with pytest.raises(_cabi.CpdError, match="sigma2"):
        _cabi.filterreg_estep(src, tgt, 0.0, False)
    with pytest.raises(_cabi.CpdError, match="non-finite"):
        _cabi.filterreg_estep(np.r_[src, [[np.nan, 0, 0]]], tgt, 0.1, False)
    with pytest.raises(_cabi.CpdError, match="d must be 2 or 3"):
        _cabi.lattice_filter(np.zeros((4, 4)), np.ones((4, 1)))
    with pytest.raises(_cabi.CpdError, match="value size"):
        _cabi.lattice_filter(np.zeros((4, 3)), np.ones((4, 9)))
    with pytest.raises(ValueError, match="2 or 3 columns"):
        filterreg.RigidFilterReg(src).registration(tgt, feature_fn=lambda x: np.c_[x, x])
    with pytest.raises(ValueError, match="Unknown objective_type"):
        filterreg.registration_filterreg(src, tgt, objective_type="pt2xx")
    with pytest.raises(RuntimeError, match="No dq3d python package"):
        filterreg.DeformableKinematicFilterReg(src)


GOLDEN = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "filterreg.npz"))


def _golden_cases():
    import sys
    import os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_filterreg as mgf
    return mgf.cases()


def test_oracle_reproduces_the_reference_fixture():
    """The unmodified reference filterreg.py (float32 Kabsch / point-to-plane, the reference's own lattice), recorded by
    tests/golden/make_golden_filterreg.py, against the FP64 oracle loop from the reference's initial sigma2."""
    for name, s, t, n, kw in _golden_cases():
        s2 = float(GOLDEN[name.split("_")[0] + "_sigma2_init"])
        init = kw.get("tf_init_params", {})
        nrm = GOLDEN["bunny_normals"] if name.startswith("bunny") else None
        rot, tt, s2o, q, it = fo.registration(s, t, nrm, s2, kw["update_sigma2"], kw.get("w", 0.0), kw["objective_type"], kw["maxiter"],
                                              kw["tol"], 1e-4, init.get("rot"), init.get("t"), impl=_impl())
        assert it == int(GOLDEN[name + "_iters"]), name
        np.testing.assert_allclose(rot, GOLDEN[name + "_rot"], rtol=0, atol=1e-5, err_msg=name)
        np.testing.assert_allclose(tt, GOLDEN[name + "_t"], rtol=0, atol=1e-5, err_msg=name)
        assert abs(s2o / GOLDEN[name + "_sigma2"] - 1) <= 1e-5, name


def _check_public_api_against_fixture():
    for name, s, t, n, kw in _golden_cases():
        calls = []
        nrm = GOLDEN["bunny_normals"] if name.startswith("bunny") else None
        res = filterreg.registration_filterreg(s, t, target_normals=nrm, callbacks=[lambda tfp: calls.append(1)], **kw)
        assert len(calls) == int(GOLDEN[name + "_iters"]), name
        np.testing.assert_allclose(res.transformation.rot, GOLDEN[name + "_rot"], rtol=0, atol=1e-5, err_msg=name)
        np.testing.assert_allclose(res.transformation.t, GOLDEN[name + "_t"], rtol=0, atol=1e-5, err_msg=name)
        assert abs(res.sigma2 / GOLDEN[name + "_sigma2"] - 1) <= 1e-5, name


def test_public_api_reproduces_the_reference_fixture_emulated(emulated):
    _check_public_api_against_fixture()


@pytest.mark.gpu
def test_public_api_reproduces_the_reference_fixture_gpu():
    _check_public_api_against_fixture()


def test_kabsch_and_pt2pl_known_answers():
    rng = np.random.default_rng(8)
    x = rng.standard_normal((50, 3))
    th = 0.7
    r = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    y = x.dot(r.T) + [0.1, -0.2, 0.3]
    w = rng.random(50) + 0.1
    for fn in (fo.kabsch, filterreg.kabsch):
        rr, tt = fn(x, y, w)
        np.testing.assert_allclose(rr, r, atol=1e-12)
        np.testing.assert_allclose(tt, [0.1, -0.2, 0.3], atol=1e-12)
    rr, tt = fo.kabsch_f32(x, y, w)
    np.testing.assert_allclose(rr, r, atol=1e-5)
    # a mirrored target: the determinant correction still returns a proper rotation
    rr, _ = fo.kabsch(x, x * [1, 1, -1], w)
    assert abs(np.linalg.det(rr) - 1.0) < 1e-12
    # zero weight: identity and zero, as kabsch.cc:20-22
    rr, tt = fo.kabsch(x, y, np.zeros(50))
    assert np.array_equal(rr, np.identity(3)) and np.array_equal(tt, np.zeros(3))
    x2 = x[:, :2]
    r2 = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    for fn in (fo.kabsch2d, filterreg.kabsch2d):
        rr, tt = fn(x2, x2.dot(r2.T) + [1.0, 2.0], w)
        np.testing.assert_allclose(rr, r2, atol=1e-12)
        np.testing.assert_allclose(tt, [1.0, 2.0], atol=1e-12)
    # point to plane: a pure translation along the normals is recovered in one solve
    n = rng.standard_normal((50, 3))
    n /= np.linalg.norm(n, axis=1)[:, None]
    tw, q = fo.compute_twist_for_pt2pl(x, x + [0.0, 0.0, 0.01], n, w)
    np.testing.assert_allclose(tw, [0, 0, 0, 0, 0, 0.01], atol=1e-12)
    tw2, q2 = filterreg.compute_twist_for_pt2pl(x, x + [0.0, 0.0, 0.01], n, w)
    np.testing.assert_allclose(tw2, tw, atol=1e-15)
    assert abs(q - q2) <= 1e-15
    twf, _ = fo.pt2pl_f32(x, x + [0.0, 0.0, 0.01], n, w)
    np.testing.assert_allclose(twf, tw, atol=1e-5)


# ---- on the H100 ----------------------------------------------------------------------------------------------------------
def _lumps(count, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((12, 3)) * 0.05
    pts = centres[rng.integers(0, 12, count)] + rng.standard_normal((count, 3)) * 0.01
    return pts


@pytest.mark.gpu
@pytest.mark.parametrize("count", [100_000, 1_000_000])
def test_full_size_loop_memory_and_rerun_gpu(count):
    """The device loop at full size: its first E-step equals the oracle's bit for bit, a second handle repeats every step bit for bit,
    and the handle holds no more device memory than DESIGN.md section 3 states."""
    src = _lumps(count, 1)
    tgt = _lumps(count, 2) + 0.01
    nrm = np.random.default_rng(3).standard_normal((count, 3))
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    s2 = max(filterreg.mu.squared_kernel_sum(src, tgt), 1e-4)
    runs = []
    for _ in range(2):
        loop = _cabi.FilterRegLoop(src, tgt, nrm, True)
        moms = [loop.step(np.identity(3), np.zeros(3), s, 0.1) for s in (s2, 1e-4)]
        runs.append((moms, loop.last_estep()))
        p, d, ch = 2 * count + 1, 3, 8
        e = p * (d + 1)
        bound = 44 * e + 8 * (d + 1) * e + 2 * 4 * ch * (e + 1) + (4 * d + 4 * ch) * p + 8 * 3 * d * p + 48 * e + 2 ** 20
        assert loop.device_bytes() <= bound, (loop.device_bytes(), bound)
    assert all(np.array_equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(_same(a, b) for a, b in zip(runs[0][1][:4], runs[1][1][:4]))
    ref = fo.expectation_step(src, tgt, 1e-4, True, nrm, impl=_impl())
    assert all(_same(a, b) for a, b in zip(runs[0][1][:4], ref[:4]))


@pytest.mark.gpu
def test_device_lattice_bit_identical_gpu():
    _check_device_lattice()


@pytest.mark.gpu
def test_estep_and_loop_gpu():
    src, tgt, nrm = _clouds(61, 1000, 3)
    _check_estep(src, tgt, nrm, 50.0, True)
    _check_estep(src, tgt, nrm, 0.05, False)
    _check_loops()
    _check_loop_edges()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [100_000, 1_000_000])
def test_full_size_estep_bit_identical_gpu(count):
    src = _lumps(count, 1)
    th = 0.2
    r = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1.0]])
    tgt = _lumps(count, 2).dot(r.T) + 0.01
    nrm = np.random.default_rng(3).standard_normal((count, 3))
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    first = max(filterreg.mu.squared_kernel_sum(src, tgt), 1e-4)
    # at 10^6 points min_sigma2 = 1e-4 still leaves fewer vertices (6 547) than n * alpha (15 000), so the lattice keeps its blur
    # there; 2e-6 (808 301 vertices) is the no-blur case at that size
    runs = [(first, True), (1e-4, count > 100_000)] + ([(2e-6, False)] if count > 100_000 else [])
    for sigma2, blur in runs:
        a = _cabi.filterreg_estep(src, tgt, sigma2, True, nrm)
        b = fo.expectation_step(src, tgt, sigma2, True, nrm, impl=_impl())
        assert a[4] == b[4] == blur
        for x, y in zip(a[:4], b[:4]):
            assert _same(x, y)
        again = _cabi.filterreg_estep(src, tgt, sigma2, True, nrm)
        for x, y in zip(a[:4], again[:4]):
            assert _same(x, y)
