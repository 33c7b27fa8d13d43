"""registration_cpd_batch / cpd_batch_register: many rigid and affine registrations in one launch, one CTA per pair.

Checked against the reference's own fixtures, the numpy oracle and the single-pair path (registration_cpd) at the parity bar
(rotation / B / translation 1e-5, sigma2 1e-6 relative, q 1e-5 relative; equal iteration counts, or one apart only where the
stop is decided inside the measured q discrepancy of the two runs, see _assert_same_stop), for independence of a pair's
result from the rest of the batch (bit for bit), and for its refusals.  The tests marked gpu run on the H100; the others run the
same library code under the CPU emulation (tests/emu) at small sizes.
"""
import numpy as np
import pytest

from conftest import load_golden
from oracle import cpd_oracle as orc
from probreg_b200 import _cabi, cpd

ROT_TOL = 1e-5
S2_TOL = 1e-6
Q_TOL = 1e-5

# the rigid / affine cases of test_cuda_parity.CASES: (fixture, tag, tf type, iterations, w, kwargs, source key, target key)
REF_CASES = [
    ("bunny.npz", "rigid10", "rigid", 10, 0.0, {}, "source", "target"),
    ("bunny.npz", "rigid10_w01", "rigid", 10, 0.1, {}, "source", "target"),
    ("bunny.npz", "rigid10_noscale", "rigid", 10, 0.0, {"update_scale": False}, "source", "target"),
    ("bunny.npz", "affine10", "affine", 10, 0.0, {}, "source", "target"),
    ("synthetic1500.npz", "rigid20", "rigid", 20, 0.0, {}, "source", "target"),
    ("synthetic1500.npz", "rigid20_outl_w", "rigid", 20, 0.2, {}, "source", "target_outl"),
    ("synthetic1500.npz", "rigid30_outl_w0", "rigid", 30, 0.0, {}, "source", "target_outl"),
    ("synthetic1500.npz", "affine20", "affine", 20, 0.0, {}, "source_a", "target_a"),
    ("nonrigid.npz", "fishaffine15", "affine", 15, 0.0, {}, "fish_source", "fish_target"),
    ("nonrigid.npz", "fishrigid15", "rigid", 15, 0.0, {}, "fish_source", "fish_target"),
]


@pytest.fixture(scope="module")
def goldens():
    return {f: load_golden(f) for f in ("bunny.npz", "synthetic1500.npz", "nonrigid.npz")}


def _rot3(rng, max_deg):
    ax = rng.standard_normal(3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(rng.uniform(0.0, max_deg))
    k = np.array([[0.0, -ax[2], ax[1]], [ax[2], 0.0, -ax[0]], [-ax[1], ax[0], 0.0]])
    return np.identity(3) + np.sin(a) * k + (1.0 - np.cos(a)) * k.dot(k)


def _rot2(deg):
    a = np.deg2rad(deg)
    return np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])


def ragged_pairs(seed, sizes, dim=3):
    """Seeded pairs: a source box, the target a rotated (<= 45 deg), shifted, noised and re-sampled copy of another draw of it."""
    rng = np.random.default_rng(seed)
    src, tgt = [], []
    for m, n in sizes:
        s = rng.random((m, dim)) * np.array([1.0, 0.6, 0.3][:dim])
        base = rng.random((n, dim)) * np.array([1.0, 0.6, 0.3][:dim])
        r = _rot3(rng, 45.0) if dim == 3 else _rot2(rng.uniform(-45.0, 45.0))
        src.append(s)
        tgt.append(base.dot(r.T) + rng.uniform(-0.1, 0.1, dim) + 0.01 * rng.standard_normal((n, dim)))
    return src, tgt


# the 8 oracle pairs: m != n, one pair with m = 1 and one with n = 1 (their rotation is undetermined: A = 0, so only sigma2 and q
# are compared there, with update_scale off), w 0 / 0.1, update_scale on / off, non-identity warm starts
ORACLE_SIZES = [(1, 120), (130, 1), (180, 60), (45, 170), (200, 140), (90, 200), (160, 75), (33, 190)]


def _oracle_batch(seed, sizes, w, update_scale, tf_type):
    src, tgt = ragged_pairs(seed, sizes)
    rng = np.random.default_rng(seed + 100)
    inits = []
    for k in range(len(src)):
        if tf_type == "rigid":
            inits.append({"rot": _rot3(rng, 10.0), "t": rng.uniform(-0.05, 0.05, 3), "scale": 1.0 + 0.05 * k})
        else:
            inits.append({"b": np.identity(3) + 0.03 * rng.standard_normal((3, 3)), "t": rng.uniform(-0.05, 0.05, 3)})
    return src, tgt, inits


def converging_pairs(seed, sizes):
    """Seeded pairs that converge under the default tol well before maxiter: source and target are random subsets of one box
    cloud, the target rotated (<= 45 deg), shifted and noised."""
    rng = np.random.default_rng(seed)
    src, tgt = [], []
    for m, n in sizes:
        base = rng.random((max(m, n), 3)) * np.array([1.0, 0.6, 0.3])
        r = _rot3(rng, 45.0)
        src.append(base[rng.permutation(base.shape[0])[:m]])
        tgt.append(base[rng.permutation(base.shape[0])[:n]].dot(r.T) + rng.uniform(-0.1, 0.1, 3) + 0.005 * rng.standard_normal((n, 3)))
    return src, tgt


CONVERGING_SIZES = [(180, 60), (200, 140), (90, 200), (160, 75), (120, 150), (397, 397)]
STOP_MAXITER = 100      # the default tol with room to stop: every pair of these tests stops before it


def _assert_same_stop(it, it_ref, q_at, q_ref_at, tol):
    """The stop rule |q - q_prev| < tol gives equal counts unless the two runs' q differ enough to move |q_k - q_(k-1)| across tol.
    Counts may differ by one only there: at k = min(it, it_ref) the reference's |q_k - q_(k-1)| must lie within the measured q
    discrepancy of the two runs at k and k - 1 (q_at / q_ref_at: q after k iterations, k = 0 the start) of tol."""
    if it == it_ref:
        return
    assert abs(int(it) - int(it_ref)) == 1, (it, it_ref)
    k = int(min(it, it_ref))
    window = abs(q_at(k) - q_ref_at(k)) + abs(q_at(k - 1) - q_ref_at(k - 1))
    dq = abs(q_ref_at(k) - q_ref_at(k - 1))
    assert abs(dq - tol) <= window, (k, dq, tol, window)


def _batch_q_at(s, t, tf_type, w, update_scale, init):
    def q_at(k):
        res, _ = cpd.registration_cpd_batch([s], [t], tf_type, w=w, maxiter=k, tol=-1.0, update_scale=update_scale,
                                            tf_init_params=[init] if init else None)
        return res[0].q
    return q_at


def _check_vs_oracle(src, tgt, inits, res, iters, tf_type, w, update_scale, maxiter, tol):
    for k, (s, t) in enumerate(zip(src, tgt)):
        ini = inits[k] if inits is not None else {}
        init = None
        if ini:
            init = (ini["rot"], ini["t"], ini["scale"]) if tf_type == "rigid" else (ini["b"], ini["t"])
        us = update_scale and s.shape[0] > 1 and t.shape[0] > 1
        s20 = orc.sigma2_init_exact(s, t)
        trace = []
        o, oit = orc.registration(s, t, tf_type, w=w, maxiter=maxiter, tol=tol, update_scale=us, init=init, sigma2_0=s20, trace=trace)
        r = res[k]
        if iters[k] != oit:
            qo = [1.0 + t.shape[0] * s.shape[1] * 0.5 * np.log(s20)] + [q for _, q in trace]
            _assert_same_stop(iters[k], oit, _batch_q_at(s, t, tf_type, w, us, ini), lambda i: qo[i], tol)
            kk = int(min(iters[k], oit))       # compare the two at the common count
            o, _ = orc.registration(s, t, tf_type, w=w, maxiter=kk, tol=-1.0, update_scale=us, init=init, sigma2_0=s20)
            rr, _ = cpd.registration_cpd_batch([s], [t], tf_type, w=w, maxiter=kk, tol=-1.0, update_scale=us,
                                               tf_init_params=[ini] if ini else None)
            r = rr[0]
        assert r.sigma2 == pytest.approx(o.sigma2, rel=S2_TOL), k
        assert r.q == pytest.approx(o.q, rel=Q_TOL), k
        if s.shape[0] > 1 and t.shape[0] > 1:
            lin = r.transformation.rot if tf_type == "rigid" else r.transformation.b
            np.testing.assert_allclose(lin, o.params[0], atol=ROT_TOL, err_msg="pair %d" % k)
            np.testing.assert_allclose(r.transformation.t, o.params[1], atol=ROT_TOL, err_msg="pair %d" % k)
        elif s.shape[0] == 1:       # one source: the rotation is undetermined, where it lands is not
            np.testing.assert_allclose(r.transformation.transform(s), orc.apply_rigid(s, *o.params), atol=ROT_TOL)


def _run_oracle_case(tf_type, w, update_scale, seed):
    src, tgt, inits = _oracle_batch(seed, ORACLE_SIZES, w, update_scale, tf_type)
    if tf_type == "affine":         # a one-point cloud leaves the affine system singular (the reference's too)
        src, tgt, inits = src[2:], tgt[2:], inits[2:]
    us = update_scale
    if tf_type == "rigid" and update_scale:   # the one-point pairs need update_scale off (0 / 0 otherwise): run them apart
        res0, it0 = cpd.registration_cpd_batch(src[:2], tgt[:2], tf_type, w=w, maxiter=12, tol=-1.0, update_scale=False,
                                               tf_init_params=inits[:2])
        _check_vs_oracle(src[:2], tgt[:2], inits[:2], res0, it0, tf_type, w, False, 12, -1.0)
        src, tgt, inits = src[2:], tgt[2:], inits[2:]
    res, iters = cpd.registration_cpd_batch(src, tgt, tf_type, w=w, maxiter=12, tol=-1.0, update_scale=us, tf_init_params=inits)
    _check_vs_oracle(src, tgt, inits, res, iters, tf_type, w, us, 12, -1.0)
    # and with the default tol on pairs that converge: iteration counts equal to the oracle's
    src, tgt = converging_pairs(seed, CONVERGING_SIZES)
    inits = _oracle_batch(seed, CONVERGING_SIZES, w, update_scale, tf_type)[2]
    res, iters = cpd.registration_cpd_batch(src, tgt, tf_type, w=w, maxiter=STOP_MAXITER, update_scale=us, tf_init_params=inits)
    assert (iters < STOP_MAXITER).sum() >= len(iters) - 1, iters       # the stop itself is exercised
    _check_vs_oracle(src, tgt, inits, res, iters, tf_type, w, us, STOP_MAXITER, 1e-3)


def _params(r):
    t = r.transformation
    lin = t.rot if isinstance(t, cpd.tf.RigidTransformation) else t.b
    return np.r_[np.ravel(lin), np.ravel(t.t), getattr(t, "scale", 1.0), r.sigma2, r.q]


def _check_independence(src, tgt):
    """A pair's outputs are bit-identical alone, in the batch, at every position of a shuffled batch, and on a rerun."""
    res, it = cpd.registration_cpd_batch(src, tgt, "rigid", w=0.05, maxiter=8, tol=-1.0)
    again, it2 = cpd.registration_cpd_batch(src, tgt, "rigid", w=0.05, maxiter=8, tol=-1.0)
    perm = np.random.default_rng(3).permutation(len(src))
    shuf, it3 = cpd.registration_cpd_batch([src[i] for i in perm], [tgt[i] for i in perm], "rigid", w=0.05, maxiter=8, tol=-1.0)
    for k in range(len(src)):
        a = _params(res[k])
        assert np.array_equal(a, _params(again[k])), k
        assert np.array_equal(a, _params(shuf[int(np.flatnonzero(perm == k)[0])])), k
    for k in (0, len(src) - 1):
        alone, _ = cpd.registration_cpd_batch([src[k]], [tgt[k]], "rigid", w=0.05, maxiter=8, tol=-1.0)
        assert np.array_equal(_params(alone[0]), _params(res[k])), k
    assert np.array_equal(it, it2)


# ---- CPU emulation ---------------------------------------------------------------------------------------------------------
def test_emulated_fish_and_bunny_vs_reference(emulated, goldens):
    g = goldens["nonrigid.npz"]
    for tag, tf_type in (("fishrigid15", "rigid"), ("fishaffine15", "affine")):
        ps, pt = ragged_pairs(5, [(60, 130), (140, 45)], dim=2)
        res, iters = cpd.registration_cpd_batch([ps[0], g["fish_source"], ps[1]], [pt[0], g["fish_target"], pt[1]], tf_type, maxiter=15,
                                                tol=-1.0)
        assert list(iters) == [15, 15, 15]
        for r in res[1:2]:
            assert r.sigma2 == pytest.approx(float(g[tag + "_sigma2"]), rel=S2_TOL)
            assert r.q == pytest.approx(float(g[tag + "_q"]), rel=Q_TOL)
            lin = r.transformation.rot if tf_type == "rigid" else r.transformation.b
            np.testing.assert_allclose(lin, g[tag + ("_rot" if tf_type == "rigid" else "_b")], atol=ROT_TOL)
            np.testing.assert_allclose(r.transformation.t, g[tag + "_t"], atol=ROT_TOL)
    b = goldens["bunny.npz"]
    res, iters = cpd.registration_cpd_batch([b["source"]], [b["target"]], "rigid", w=0.1, maxiter=10, tol=-1.0)
    assert res[0].sigma2 == pytest.approx(float(b["rigid10_w01_sigma2"]), rel=S2_TOL)
    np.testing.assert_allclose(res[0].transformation.rot, b["rigid10_w01_rot"], atol=ROT_TOL)
    np.testing.assert_allclose(res[0].transformation.t, b["rigid10_w01_t"], atol=ROT_TOL)


@pytest.mark.parametrize("tf_type,w,update_scale", [("rigid", 0.0, True), ("rigid", 0.1, False), ("affine", 0.1, True)])
def test_emulated_vs_oracle(emulated, tf_type, w, update_scale):
    _run_oracle_case(tf_type, w, update_scale, seed=11)


def test_emulated_independence_bit_for_bit(emulated):
    src, tgt = ragged_pairs(21, [(60, 90), (150, 40), (7, 33), (120, 120), (200, 17)])
    _check_independence(src, tgt)


def test_emulated_2d_and_maxiter_zero(emulated):
    src, tgt = ragged_pairs(4, [(50, 70), (80, 30)], dim=2)
    res, iters = cpd.registration_cpd_batch(src, tgt, "rigid", maxiter=10, tol=-1.0)
    for k in range(2):
        o, _ = orc.registration(src[k], tgt[k], "rigid", maxiter=10, tol=-1.0, sigma2_0=orc.sigma2_init_exact(src[k], tgt[k]))
        assert res[k].sigma2 == pytest.approx(o.sigma2, rel=S2_TOL)
        np.testing.assert_allclose(res[k].transformation.rot, o.params[0], atol=ROT_TOL)
        np.testing.assert_allclose(res[k].transformation.t, o.params[1], atol=ROT_TOL)
    res, iters = cpd.registration_cpd_batch(src, tgt, "affine", maxiter=0)
    assert list(iters) == [0, 0]
    for k in range(2):
        s2 = orc.sigma2_init_exact(src[k], tgt[k])
        assert res[k].sigma2 == pytest.approx(s2, rel=1e-12)
        assert res[k].q == pytest.approx(1.0 + tgt[k].shape[0] * 2 * 0.5 * np.log(s2), rel=1e-12)
        np.testing.assert_array_equal(res[k].transformation.b, np.identity(2))


def test_refusals(emulated):
    src, tgt = ragged_pairs(2, [(20, 30), (25, 35), (30, 20)])
    with pytest.raises(ValueError, match="same length"):
        cpd.registration_cpd_batch(src, tgt[:2])
    with pytest.raises(ValueError, match="pair 1"):
        cpd.registration_cpd_batch([src[0], src[1][:, :2], src[2]], tgt)
    with pytest.raises(ValueError, match="registration_cpd"):
        cpd.registration_cpd_batch(src, tgt, "nonrigid")
    with pytest.raises(ValueError, match="Unknown transformation type"):
        cpd.registration_cpd_batch(src, tgt, "similarity")
    with pytest.raises(_cabi.CpdError, match="pair 2: the target is empty"):
        cpd.registration_cpd_batch(src, [tgt[0], tgt[1], np.zeros((0, 3))])
    bad = src[1].copy()
    bad[3, 1] = np.nan
    with pytest.raises(_cabi.CpdError, match="pair 1: the source has a non-finite coordinate"):
        cpd.registration_cpd_batch([src[0], bad, src[2]], tgt)
    with pytest.raises(_cabi.CpdError, match=r"w must be in \[0, 1\)"):
        cpd.registration_cpd_batch(src, tgt, w=1.0)
    big = np.random.default_rng(0).random((8193, 3))
    with pytest.raises(_cabi.CpdError, match="pair 1: m n = 8193 x 8193 exceeds .*registration_cpd"):
        cpd.registration_cpd_batch([src[0], big], [tgt[0], big])
    with pytest.raises(_cabi.CpdError, match="pair 1: 70000 sources and 1 targets: .*2\\^16 points per cloud"):
        cpd.registration_cpd_batch([src[0], np.random.default_rng(1).random((70000, 3))], [tgt[0], tgt[0][:1]])
    with pytest.raises(_cabi.CpdError, match="pair 0: sigma2_0 = 0"):
        cpd.registration_cpd_batch([np.ones((4, 3))], [np.ones((5, 3))])
    with pytest.raises(ValueError, match="pair 0: unknown tf_init_params"):
        cpd.registration_cpd_batch(src, tgt, tf_init_params=[{"b": np.identity(3)}, None, None])


# ---- H100 ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reference_fixture_cases_in_batches(goldens):
    groups = {}
    for case in REF_CASES:
        fname, tag, tf_type, iters, w, kw, sk, tk = case
        groups.setdefault((tf_type, w, tuple(sorted(kw.items())), iters), []).append(case)
    for (tf_type, w, kw, iters), cases in groups.items():
        src = [goldens[c[0]][c[6]] for c in cases]
        tgt = [goldens[c[0]][c[7]] for c in cases]
        # each group inside a batch of unrelated ragged pairs of the same D, before and after the fixtures
        dim = src[0].shape[1]
        ps, pt = ragged_pairs(len(src) + 7 * dim, [(250, 180), (70, 400), (333, 90)], dim=dim)
        src, tgt = ps[:2] + src + ps[2:], pt[:2] + tgt + pt[2:]
        res, its = cpd.registration_cpd_batch(src, tgt, tf_type, w=w, maxiter=iters, tol=-1.0, **dict(kw))
        assert all(i == iters for i in its)
        for k, c in enumerate(cases):
            g, tag = goldens[c[0]], c[1]
            r = res[k + 2]
            assert r.sigma2 == pytest.approx(float(g[tag + "_sigma2"]), rel=S2_TOL), tag
            assert r.q == pytest.approx(float(g[tag + "_q"]), rel=Q_TOL), tag
            if tf_type == "rigid":
                np.testing.assert_allclose(r.transformation.rot, g[tag + "_rot"], atol=ROT_TOL, err_msg=tag)
                assert r.transformation.scale == pytest.approx(float(g[tag + "_scale"]), rel=ROT_TOL)
            else:
                np.testing.assert_allclose(r.transformation.b, g[tag + "_b"], atol=ROT_TOL, err_msg=tag)
            np.testing.assert_allclose(r.transformation.t, g[tag + "_t"], atol=ROT_TOL, err_msg=tag)


@pytest.mark.gpu
@pytest.mark.parametrize("tag,tf_type", [("rigid_default", "rigid"), ("affine_default", "affine")])
def test_default_tolerance_stops_where_the_reference_does(goldens, tag, tf_type):
    b, s = goldens["bunny.npz"], goldens["synthetic1500.npz"]
    src = [s["source"], b["source"], orc.synthetic_pair(700, seed=3)[0]]
    tgt = [s["target"], b["target"], orc.synthetic_pair(700, seed=3)[1]]
    res, iters = cpd.registration_cpd_batch(src, tgt, tf_type)
    assert iters[1] == int(b[tag + "_iters"])
    assert res[1].sigma2 == pytest.approx(float(b[tag + "_sigma2"]), rel=S2_TOL)
    if tf_type == "rigid":
        np.testing.assert_allclose(res[1].transformation.rot, orc.rot_z(30.0), atol=ROT_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("tf_type,w,update_scale", [("rigid", 0.0, True), ("rigid", 0.1, False), ("affine", 0.0, True),
                                                    ("affine", 0.1, True)])
def test_vs_oracle(tf_type, w, update_scale):
    _run_oracle_case(tf_type, w, update_scale, seed=31)


def _check_vs_single(src, tgt, res, iters, tf_type, maxiter, tol, **kw):
    for k, (s, t) in enumerate(zip(src, tgt)):
        one = cpd.registration_cpd(s, t, tf_type, maxiter=maxiter, tol=tol, **kw)
        r = res[k]
        if tol >= 0:
            n_it = [0]
            cpd.registration_cpd(s, t, tf_type, maxiter=maxiter, tol=tol, callbacks=[lambda _: n_it.__setitem__(0, n_it[0] + 1)], **kw)
            if iters[k] != n_it[0]:
                def single_q_at(i):
                    if i == 0:
                        return 1.0 + t.shape[0] * s.shape[1] * 0.5 * np.log(cpd.RigidCPD(s)._squared_kernel_sum(s, t))
                    return cpd.registration_cpd(s, t, tf_type, maxiter=i, tol=-1.0, **kw).q
                _assert_same_stop(iters[k], n_it[0], _batch_q_at(s, t, tf_type, kw.get("w", 0.0), True, None), single_q_at, tol)
                kk = int(min(iters[k], n_it[0]))       # compare the two at the common count
                one = cpd.registration_cpd(s, t, tf_type, maxiter=kk, tol=-1.0, **kw)
                r = cpd.registration_cpd_batch([s], [t], tf_type, maxiter=kk, tol=-1.0, **kw)[0][0]
        assert r.sigma2 == pytest.approx(one.sigma2, rel=S2_TOL), k
        assert r.q == pytest.approx(one.q, rel=Q_TOL), k
        lin, lin1 = (r.transformation.rot, one.transformation.rot) if tf_type == "rigid" else (r.transformation.b, one.transformation.b)
        np.testing.assert_allclose(lin, lin1, atol=ROT_TOL, err_msg="pair %d" % k)
        np.testing.assert_allclose(r.transformation.t, one.transformation.t, atol=ROT_TOL, err_msg="pair %d" % k)


@pytest.mark.gpu
@pytest.mark.parametrize("tf_type", ["rigid", "affine"])
def test_vs_single_path_default_tol(tf_type):
    src, tgt = converging_pairs(41, CONVERGING_SIZES + [(1500, 1100)])
    res, iters = cpd.registration_cpd_batch(src, tgt, tf_type, w=0.05, maxiter=STOP_MAXITER)
    assert (iters < STOP_MAXITER).sum() >= len(iters) - 1, iters       # the stop itself is exercised
    _check_vs_single(src, tgt, res, iters, tf_type, STOP_MAXITER, 1e-3, w=0.05)


@pytest.mark.gpu
def test_independence_bit_for_bit():
    rng = np.random.default_rng(8)
    src, tgt = ragged_pairs(9, [(int(a), int(b)) for a, b in rng.integers(200, 2500, (40, 2))])
    _check_independence(src, tgt)


@pytest.mark.gpu
def test_user_sizes_1024_pairs():
    import torch

    rng = np.random.default_rng(2024)
    sizes = [(int(a), int(b)) for a, b in rng.integers(200, 4001, (1024, 2))]
    src, tgt = ragged_pairs(77, sizes)
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info(0)[0]
    res, iters = cpd.registration_cpd_batch(src, tgt, "rigid", w=0.02, maxiter=30, tol=-1.0)
    assert torch.cuda.mem_get_info(0)[0] == free0          # the call leaves nothing allocated
    assert (iters == 30).all()
    sample = rng.choice(1024, 8, replace=False)
    _check_vs_oracle([src[k] for k in sample], [tgt[k] for k in sample], None, [res[k] for k in sample], iters[sample], "rigid", 0.02,
                     True, 30, -1.0)
    _check_vs_single(src, tgt, res, iters, "rigid", 30, -1.0, w=0.02)
