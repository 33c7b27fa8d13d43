"""GMMTree (cpd_gmmtree_*, probreg_b200.gmmtree): the tree build and the registration E-step on the device.

  1. known answers: 8 anisotropic clusters far apart, L = 1, one seed per cluster -- every node is its cluster's (N_c / N, mean,
     population covariance); the same clusters under a small known motion -- registration recovers it;
  2. the build against the float64 oracle (oracle/gmmtree_oracle.py) from the same leaf seeds: iterations per level, the final
     argmax of every point, node parameters within 1e-9 of the level's largest magnitude;
  3. the registration E-step against the oracle on installed trees (far outlier, det < 1e-15, a dead node, lambda_c = 1 and 0);
  4. the full registration against the oracle over 20 iterations: rot, t and q per iteration;
  5. the refusals and the Python surface;
  6. (GPU) items 2-4 at 20 000 points; 1M points at L = 3, bit-identical twice, with the device memory it takes.
CPU tests run under the emulation of tests/emu (a few hundred points); the gpu-marked ones on the H100.
"""
import numpy as np
import pytest

from oracle import gmmtree_oracle as go
from probreg_b200 import _cabi, gmmtree

REL = 1e-9


def _rot(axis, deg):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.identity(3) + np.sin(th) * k + (1.0 - np.cos(th)) * k.dot(k)


def _clusters(per=40, seed=0):
    """8 clusters at the corners of a cube of edge 40, widths (1, 0.5, 0.25) in a random frame each; (points, first index of each
    cluster, labels)"""
    rng = np.random.default_rng(seed)
    pts, first, lab = [], [], []
    for c, corner in enumerate([(x, y, z) for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)]):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        n = per + 3 * c
        first.append(sum(len(p) for p in pts))
        pts.append(20.0 * np.array(corner) + (rng.standard_normal((n, 3)) * [1.0, 0.5, 0.25]).dot(q.T))
        lab += [c] * n
    return np.concatenate(pts), np.array(first), np.array(lab)


def _synthetic(n, seed=0):
    """an anisotropic blob cloud: a few Gaussian lumps of different shapes"""
    rng = np.random.default_rng(seed)
    k = 5
    centres = rng.uniform(-1.0, 1.0, (k, 3))
    scales = rng.uniform(0.05, 0.3, (k, 3))
    lab = rng.integers(0, k, n)
    return centres[lab] + rng.standard_normal((n, 3)) * scales[lab]


def _stack(nodes):
    return (np.array([n[0] for n in nodes]), np.array([n[1] for n in nodes]), np.array([n[2] for n in nodes]))


def _moments_array(mom):
    return np.array([np.concatenate([[m[0]], m[1], np.asarray(m[2]).ravel()]) for m in mom])


def _bunny(bunny):
    return np.ascontiguousarray(bunny["source"])


# ---- 1. known answers ---------------------------------------------------------------------------------------------------------------
def _check_clusters():
    pts, first, lab = _clusters()
    n = len(pts)
    h = _cabi.Handle(3)
    h.set_source(pts)
    h.gmmtree_build(1, 1e-3, 1e-4, first)
    pi, mu, cov = h.gmmtree_nodes()
    onodes, _, _, _ = go.build(pts, 1, 1e-3, 1e-4, first)
    for c in range(8):
        p = pts[lab == c]
        d = p - p.mean(0)
        want = (len(p) / n, p.mean(0), d.T.dot(d) / len(p))
        for got in ((pi[c], mu[c], cov[c]), onodes[c]):
            assert abs(got[0] - want[0]) <= 1e-12
            np.testing.assert_allclose(got[1], want[1], rtol=0, atol=1e-12 * 20)
            np.testing.assert_allclose(got[2], want[2], rtol=0, atol=1e-12)
    assert (h.gmmtree_assign() == lab).all()


def _check_known_motion():
    pts, first, _ = _clusters()
    rot, t = _rot([1.0, 2.0, 0.5], 2.0), np.array([0.2, -0.1, 0.15])
    tgt = pts.dot(rot.T) + t
    gt = gmmtree.GMMTree(pts, tree_level=1)
    gt.leaf_seeds = first
    gt._h.gmmtree_build(1, 1e-3, 1e-4, first)
    gt._set_nodes(*gt._h.gmmtree_nodes())
    res = gt.registration(tgt, maxiter=20, tol=-1.0)
    np.testing.assert_allclose(res.transformation.rot, rot, atol=1e-6)
    np.testing.assert_allclose(res.transformation.t, t, atol=1e-6)


# ---- 2. the build against the oracle ------------------------------------------------------------------------------------------------
def _check_build(pts, levels, seed, maxiter=1000):
    seeds = np.random.default_rng(seed).integers(0, len(pts), 8 ** levels)
    h = _cabi.Handle(3)
    h.set_source(pts)
    iters = h.gmmtree_build(levels, 1e-3, 1e-4, seeds, maxiter)
    pi, mu, cov = h.gmmtree_nodes()
    onodes, oiters, ocur, _ = go.build(pts, levels, 1e-3, 1e-4, seeds, maxiter)
    assert list(iters) == oiters
    assert (h.gmmtree_assign() == ocur).all()
    opi, omu, ocov = _stack(onodes)
    worst = 0.0
    for l in range(levels):
        s = slice(go.level(l), go.level(l + 1))
        for a, b in ((pi[s], opi[s]), (mu[s], omu[s]), (cov[s], ocov[s])):
            scale = max(np.abs(b).max(), 1e-300)
            err = np.abs(a - b).max() / scale
            worst = max(worst, err)
            assert err <= REL, (l, err)
    print("build L=%d seed=%d m=%d iters=%s worst relative error %.3g" % (levels, seed, len(pts), list(iters), worst))
    return onodes


# ---- 3. the registration E-step on installed trees ----------------------------------------------------------------------------------
def _special_tree(pts, levels, seed):
    onodes, _, _, _ = go.build(pts, levels, 1e-3, 1e-4, np.random.default_rng(seed).integers(0, len(pts), 8 ** levels), 30)
    nodes = list(onodes)
    last = go.level(levels - 1)
    nodes[last + 1] = (0.0, np.zeros(3), np.identity(3))                    # a dead node
    pi, mu, _ = nodes[last + 2]
    nodes[last + 2] = (pi, mu, 1e-6 * np.identity(3))                        # det 1e-18 < 1e-15: pdf 0
    if levels > 1:
        pi, mu, _ = nodes[3]
        nodes[3] = (pi, mu, np.diag([1e-7, 1.0, 1.0]) * 1e-2)                # det < 1e-15 on an inner node too
    return nodes


def _check_estep(pts, tgt, levels, seed):
    nodes = _special_tree(pts, levels, seed)
    h = _cabi.Handle(3)
    h.set_target(tgt)
    h.gmmtree_load(levels, *_stack(nodes))
    rot, t = _rot([0.3, -1.0, 0.2], 5.0), np.array([0.01, 0.02, -0.03])
    for lambda_c in (0.0, 0.01, 0.05, 1.0):
        mom = h.gmmtree_estep(rot, t, lambda_c)
        ref = _moments_array(go.reg_estep(tgt.dot(rot.T) + t, nodes, levels, lambda_c))
        err = np.abs(mom - ref).max() / np.abs(ref).max()
        assert err <= REL, (lambda_c, err)
        if lambda_c == 1.0:                       # everything stops at level 0
            assert np.all(mom[8:, 0] == 0.0)
        if lambda_c == 0.0:                       # everything descends to the leaves (no node here has complexity <= 0)
            assert np.all(mom[: go.level(levels - 1), 0] == 0.0)
    return mom


def _estep_target(pts, seed):
    rng = np.random.default_rng(seed)
    tgt = pts[rng.permutation(len(pts))[: len(pts) // 2]] + 0.01 * rng.standard_normal((len(pts) // 2, 3))
    tgt[0] = [1e6, -1e6, 1e6]                     # a far outlier: gamma all 0, child 0 all the way down
    return np.ascontiguousarray(tgt)


# ---- 4. the full registration -------------------------------------------------------------------------------------------------------
class _Recording(gmmtree.GMMTree):
    def maximization_step(self, estep_res, trans_p):
        res = super(_Recording, self).maximization_step(estep_res, trans_p)
        self.trace.append(res.q)
        return res


def _check_registration(pts, levels, seed, maxiter=20):
    tgt = pts.dot(_rot([0.2, 0.4, 1.0], 10.0).T) + np.array([0.02, -0.01, 0.03])
    gt = _Recording(pts, tree_level=levels, seed=seed)
    gt.trace = []
    res = gt.registration(tgt, maxiter=maxiter, tol=-1.0)
    onodes = [(n[0], n[1], n[2]) for n in gt._nodes]          # the device's tree: the loop is compared on the same one
    orot, ot, _, otrace = go.registration(onodes, tgt, levels, 0.01, maxiter, -1.0)
    np.testing.assert_allclose(res.transformation.rot, orot, atol=1e-8)
    np.testing.assert_allclose(res.transformation.t, ot, atol=1e-8)
    np.testing.assert_allclose(gt.trace, otrace, rtol=REL)
    return res


# ---- 5. refusals and the Python surface ---------------------------------------------------------------------------------------------
def _check_refusals():
    pts = _synthetic(300, 3)
    seeds = np.arange(64) % len(pts)
    h2 = _cabi.Handle(2)
    h2.set_source(pts[:, :2])
    with pytest.raises(_cabi.CpdError, match="3-D"):
        h2.gmmtree_build(1, 1e-3, 1e-4, seeds[:8])
    h = _cabi.Handle(3)
    with pytest.raises(_cabi.CpdError, match="source"):
        h.gmmtree_build(1, 1e-3, 1e-4, seeds[:8])
    h.set_source(pts)
    for lv in (0, 6):
        with pytest.raises(ValueError):
            h.gmmtree_build(lv, 1e-3, 1e-4, seeds)
        with pytest.raises(_cabi.CpdError, match="tree_level"):
            _cabi.check(h._lib.cpd_gmmtree_build(h._h, lv, 1e-3, 1e-4, seeds.ctypes.data_as(_cabi.ctypes.POINTER(_cabi.ctypes.c_int64)),
                                                 10, None))
    for bad in (-1, len(pts)):
        s = seeds[:8].copy()
        s[5] = bad
        with pytest.raises(_cabi.CpdError, match="seed"):
            h.gmmtree_build(1, 1e-3, 1e-4, s)
    with pytest.raises(_cabi.CpdError, match="finite"):
        h.gmmtree_build(1, float("nan"), 1e-4, seeds[:8])
    with pytest.raises(_cabi.CpdError, match="maxiter"):
        h.gmmtree_build(1, 1e-3, 1e-4, seeds[:8], 0)
    with pytest.raises(_cabi.CpdError, match="no GMMTree"):
        h.gmmtree_estep(np.identity(3), np.zeros(3), 0.01)
    with pytest.raises(_cabi.CpdError, match="no GMMTree"):
        h.gmmtree_nodes()
    bad_pts = pts.copy()
    bad_pts[7, 1] = np.inf
    hb = _cabi.Handle(3)
    hb.set_source(bad_pts)
    with pytest.raises(_cabi.CpdError, match="non-finite"):
        hb.gmmtree_build(1, 1e-3, 1e-4, seeds[:8])
    h.gmmtree_build(1, 1e-3, 1e-4, seeds[:8], 5)
    with pytest.raises(_cabi.CpdError, match="target"):
        h.gmmtree_estep(np.identity(3), np.zeros(3), 0.01)
    h.set_target(pts)
    for r, t, lc in ((np.full((3, 3), np.nan), np.zeros(3), 0.01), (np.identity(3), [0, np.inf, 0], 0.01),
                     (np.identity(3), np.zeros(3), float("nan"))):
        with pytest.raises(_cabi.CpdError, match="finite"):
            h.gmmtree_estep(r, t, lc)
    pi, mu, cov = h.gmmtree_nodes()
    cov[3, 0, 0] = np.nan
    with pytest.raises(_cabi.CpdError, match="non-finite"):
        h.gmmtree_load(1, pi, mu, cov)
    # the tree survives a new source; the assignments do not survive a new source count
    h.gmmtree_build(1, 1e-3, 1e-4, seeds[:8], 5)
    before = h.gmmtree_nodes()
    h.set_source(pts[:200])
    for a, b in zip(before, h.gmmtree_nodes()):
        np.testing.assert_array_equal(a, b)
    h.gmmtree_estep(np.identity(3), np.zeros(3), 0.01)
    with pytest.raises(_cabi.CpdError, match="changed"):
        h.gmmtree_assign()
    h.gmmtree_load(1, *before)
    with pytest.raises(_cabi.CpdError, match="built"):
        h.gmmtree_assign()


def _check_comm_refused():
    pts = _synthetic(100, 4)
    uid = _cabi.unique_id()
    comm = _cabi.comm_create(0, 1, 0, uid)
    try:
        h = _cabi.Handle(3)
        h.set_source(pts)
        h.set_target(pts)
        h.attach_comm(comm, 1, 0)
        with pytest.raises(_cabi.CpdError, match="communicator"):
            h.gmmtree_build(1, 1e-3, 1e-4, np.arange(8))
        with pytest.raises(_cabi.CpdError, match="communicator"):
            h.gmmtree_load(1, np.full(8, 0.125), np.zeros((8, 3)), np.tile(np.identity(3), (8, 1, 1)))
        h.close()
    finally:
        _cabi.comm_destroy(comm)


def _check_surface():
    pts = _synthetic(300, 5)
    tgt = pts.dot(_rot([0, 0, 1], 5.0).T)
    gt = gmmtree.GMMTree(pts, tree_level=2, seed=3, build_maxiter=7)
    assert len(gt._nodes) == 72
    for pi, mu, cov in gt._nodes:
        assert np.ndim(pi) == 0 and np.shape(mu) == (3,) and np.shape(cov) == (3, 3)
    np.testing.assert_array_equal(gt.leaf_seeds, np.random.default_rng(3).integers(0, 300, 64))
    assert len(gt.build_iterations) == 2 and max(gt.build_iterations) <= 7
    es = gt.expectation_step(tgt)
    assert len(es.moments) == 72 and np.shape(es.moments[0][2]) == (3, 3)
    assert abs(sum(m[0] for m in es.moments)) <= len(tgt)
    seen = []
    gt.set_callbacks([lambda tf: seen.append(tf)])
    res = gt.registration(tgt, maxiter=4, tol=-1.0)
    assert len(seen) == 4
    inv = gt._tf_result.inverse()
    np.testing.assert_array_equal(seen[-1].rot, inv.rot)
    np.testing.assert_array_equal(seen[-1].t, inv.t)
    np.testing.assert_array_equal(res.transformation.rot, inv.rot)
    # keyword pass-through
    r2 = gmmtree.registration_gmmtree(pts, tgt, maxiter=3, tol=-1.0, tree_level=1, seed=3, build_maxiter=4, lambda_c=0.02)
    gt1 = gmmtree.GMMTree(pts, tree_level=1, seed=3, build_maxiter=4, lambda_c=0.02)
    r1 = gt1.registration(tgt, maxiter=3, tol=-1.0)
    np.testing.assert_array_equal(r1.transformation.rot, r2.transformation.rot)
    assert r1.q == r2.q or (np.isnan(r1.q) and np.isnan(r2.q))

    # a subclass's expectation_step is driven with the moved target
    class Sub(gmmtree.GMMTree):
        calls = 0

        def expectation_step(self, target):
            Sub.calls += 1
            return super(Sub, self).expectation_step(target)

    gs = Sub(pts, tree_level=2, seed=3, build_maxiter=7)
    rs = gs.registration(tgt, maxiter=4, tol=-1.0)
    assert Sub.calls == 4
    np.testing.assert_allclose(rs.transformation.rot, res.transformation.rot, atol=1e-12)
    # set_source rebuilds
    gt.set_source(pts[:150])
    assert len(gt.leaf_seeds) == 64 and gt.leaf_seeds.max() < 150


# ---- CPU: the emulation -------------------------------------------------------------------------------------------------------------
def test_clusters_give_their_own_moments_emulated(emulated):
    _check_clusters()


def test_known_motion_is_recovered_emulated(emulated):
    _check_known_motion()


@pytest.mark.parametrize("levels,seed", [(1, 0), (1, 1), (2, 0), (2, 7)])
def test_build_matches_oracle_synthetic_emulated(emulated, levels, seed):
    _check_build(_synthetic(400, seed), levels, seed)


def test_build_matches_oracle_level3_emulated(emulated):
    _check_build(_synthetic(300, 11), 3, 11, maxiter=6)


@pytest.mark.parametrize("levels", [1, 2])
def test_build_matches_oracle_bunny_emulated(emulated, bunny, levels):
    _check_build(_bunny(bunny), levels, 5)


@pytest.mark.parametrize("levels", [1, 2, 3])
def test_estep_matches_oracle_on_installed_trees_emulated(emulated, levels):
    pts = _synthetic(400, 20 + levels)
    _check_estep(pts, _estep_target(pts, levels), levels, levels)


def test_registration_matches_oracle_bunny_emulated(emulated, bunny):
    _check_registration(_bunny(bunny), 2, 0)


def test_registration_matches_oracle_synthetic_emulated(emulated):
    _check_registration(_synthetic(400, 30), 1, 1)


def test_refusals_emulated(emulated):
    _check_refusals()


def test_communicator_refused_emulated(emulated):
    _check_comm_refused()


def test_python_surface_emulated(emulated):
    _check_surface()


def test_se3_op_matches_rodrigues():
    from probreg_b200 import se3_op

    tw = np.array([0.1, -0.2, 0.3, 1.0, 2.0, 3.0])
    rot, t = se3_op.twist_trans(tw)
    np.testing.assert_allclose(rot, _rot(tw[:3], np.rad2deg(np.linalg.norm(tw[:3]))), atol=1e-14)
    np.testing.assert_array_equal(t, tw[3:])
    r2, t2 = se3_op.twist_mul(tw, np.identity(3), np.zeros(3))
    np.testing.assert_allclose(r2, rot, atol=1e-15)
    np.testing.assert_allclose(t2, tw[3:], atol=1e-15)
    np.testing.assert_array_equal(se3_op.twist_trans(np.zeros(6))[0], np.identity(3))


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clusters_gpu():
    _check_clusters()
    _check_known_motion()


@pytest.mark.gpu
@pytest.mark.parametrize("levels,maxiter", [(1, 1000), (2, 1000), (3, 12)])
def test_build_matches_oracle_gpu(levels, maxiter):
    _check_build(_synthetic(20000, levels), levels, levels, maxiter)


@pytest.mark.gpu
def test_build_matches_oracle_bunny_gpu(bunny):
    for levels in (1, 2, 3):
        _check_build(_bunny(bunny), levels, 9)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [1, 2, 3])
def test_estep_matches_oracle_gpu(levels):
    pts = _synthetic(20000, 40 + levels)
    _check_estep(pts, _estep_target(pts, levels), levels, levels)


@pytest.mark.gpu
def test_registration_matches_oracle_gpu(bunny):
    _check_registration(_bunny(bunny), 2, 0)
    _check_registration(_synthetic(20000, 50), 2, 2)


@pytest.mark.gpu
def test_refusals_gpu():
    _check_refusals()
    _check_surface()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_million_points_level3_reproducible_gpu():
    import torch

    pts = _synthetic(1_000_000, 60)
    tgt = pts.dot(_rot([1.0, 1.0, 0.0], 3.0).T) + 0.01
    out = []
    for _ in range(2):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        gt = gmmtree.GMMTree(pts, tree_level=3, seed=1)
        res = gt.registration(tgt, maxiter=20, tol=-1.0)
        used = free0 - torch.cuda.mem_get_info(0)[0]
        print("1M points, L=3: build iterations %s, handle device memory %.1f MB" % (list(gt.build_iterations), used / 2 ** 20))
        out.append((_stack(gt._nodes), res.transformation.rot, res.transformation.t, res.q, gt._h.gmmtree_assign()))
        gt._h.close()
    (a, b) = out
    for x, y in zip(a[0], b[0]):
        np.testing.assert_array_equal(x, y)
    for x, y in zip(a[1:], b[1:]):
        np.testing.assert_array_equal(x, y)
