"""BASELINE.json configurations 3 and 4 at full size through size-independent properties (no oracle can hold them):
   3. affine CPD, N = M = 250k on one GPU;   4. rigid CPD, N = M = 1M sharded over 8 GPUs -> here ONE rank's shard
   (1M sources x 125k targets, the global N in the outlier constant), which is what each of the 8 processes executes.
Config 3 needs ~300 iterations at 250k, not the ~100 of a 3000-point cloud: EM anneals sigma2 more
slowly the denser the cloud is (3k points converge by iteration 75,
30k by 175, 250k by ~350; the 3k trajectory is the oracle's).
"""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import cpd_oracle as orc
from probreg_b200 import _cabi, cpd

def _config3(n, iters, sample):
    src, tgt = orc.synthetic_pair(n, "affine")
    seen = []
    res = cpd.registration_cpd(src, tgt, "affine", maxiter=iters, tol=-1.0, callbacks=[lambda t: seen.append(1)])
    assert len(seen) == iters
    lin = orc.rot_z(30.0).dot(np.diag([1.1, 0.9, 1.05]))
    lin[0, 1] += 0.05
    np.testing.assert_allclose(res.transformation.b, lin, atol=1e-2)
    np.testing.assert_allclose(res.transformation.t, [0.1, -0.2, 0.3], atol=1e-2)
    assert 5e-5 < res.sigma2 < 5e-3
    # one E-step at the final transform: conservation laws + a column sample against the C oracle
    ts = res.transformation.transform(src)
    es = cpd.AffineCPD(src).expectation_step(ts, tgt, res.sigma2, 0.1)
    assert es.n_p == pytest.approx(es.pt1.sum(), rel=1e-7)
    np.testing.assert_allclose(es.px.sum(0), (es.pt1[:, None] * tgt).sum(0), rtol=1e-6)
    sel = np.random.default_rng(2).choice(n, sample, replace=False)
    ref = c_oracle.expectation_step(ts, tgt[sel], res.sigma2, 0.1, n_global=n)
    np.testing.assert_allclose(es.pt1[sel], ref.pt1, rtol=5e-5, atol=1e-12)


def _config4(m, n_global, ranks, sample):
    src, tgt = orc.synthetic_pair(m)
    lo, hi = 3 * (n_global // ranks), 4 * (n_global // ranks)               # the shard rank 3 would hold
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(tgt[lo:hi], n_global=n_global, frame_origin=tgt.mean(0))
    ts = orc.apply_rigid(src, orc.rot_z(29.5), np.array([0.1, -0.2, 0.3]))
    pt1, p1, px, n_p = h.estep(ts, 3e-4, 0.1)
    assert pt1.shape == (hi - lo,) and p1.shape == (m,)
    assert n_p == pytest.approx(pt1.sum(), rel=1e-7)                          # sum_m p1 == sum_n pt1 over the shard
    np.testing.assert_allclose(px.sum(0), (pt1[:, None] * tgt[lo:hi]).sum(0), rtol=1e-6)
    sel = np.random.default_rng(3).choice(hi - lo, sample, replace=False)
    ref = c_oracle.expectation_step(ts, tgt[lo:hi][sel], 3e-4, 0.1, n_global=n_global)
    np.testing.assert_allclose(pt1[sel], ref.pt1, rtol=5e-5, atol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_config3_affine_250k_properties():
    _config3(250000, 300, 600)           # |B - B*| 3.0e-3, sigma2 1.03e-4 after 300 iterations


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_config4_one_rank_shard_of_1m():
    _config4(1000000, 1000000, 8, 300)


def test_config3_and_config4_bodies_at_emulation_size(emulated):
    """The same two test bodies at sizes the CPU emulation can run: checks the test logic itself before its first hardware run."""
    _config3(2000, 100, 150)
    _config4(4000, 4000, 8, 80)
