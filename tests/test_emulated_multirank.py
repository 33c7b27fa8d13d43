"""The target-sharded multi-rank path on the CPU: ranks are threads, each with its own handle and "device" of
the emulated library (tests/emu), and ncclAllReduce is an in-process rendezvous (tests/emu/emu_nccl.h).  What runs for real: the
shard bounds / global N / common frame origin, the per-shard E-step, the moments all-reduce + replicated M-step of the rigid and
affine loops, the M-sized all-reduces of cpd_estep, the non-rigid (dense, low-rank, constrained) paths -- compared with the
single-rank oracle and required to be bit-identical across ranks.  Not covered: the NVLink peer-memory exchange kernel (needs
cudaIpc; the Communicator falls back to the all-reduce path exactly as it does when peers cannot map each other)."""
import threading

import numpy as np
import pytest

from oracle import cpd_oracle as orc
from probreg_b200 import cpd
from probreg_b200 import dist as pdist


def _run_ranks(world, body):
    """Run body(comm) on `world` threads; returns the list of results in rank order (re-raises the first failure)."""
    barrier = threading.Barrier(world)
    box, gbox = {}, [None] * world
    results, errors = [None] * world, [None] * world

    def make(rank):
        def exchange(obj):
            if rank == 0:
                box["v"] = obj
            barrier.wait()
            v = box["v"]
            barrier.wait()
            return v

        def gather(obj):
            gbox[rank] = obj
            barrier.wait()
            out = list(gbox)
            barrier.wait()
            return out

        def run():
            try:
                comm = pdist.Communicator(rank, world, device=rank, exchange=exchange, gather=gather, use_p2p=False)
                results[rank] = body(comm)
            except BaseException as e:          # noqa: BLE001 -- reported below; do not leave the other ranks waiting
                errors[rank] = e
                barrier.abort()

        return threading.Thread(target=run)

    threads = [make(r) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=900)
    for e in errors:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in errors:
        if e is not None:
            raise e
    return results


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_estep_and_registration(emulated, monkeypatch, world):
    monkeypatch.setenv("CPD_EMU_DEVICES", str(world))
    src, tgt = orc.synthetic_pair(700)
    outl = (np.random.default_rng(3).random((41, 3)) - 0.5) * 3 + tgt.mean(0)
    tgt = np.ascontiguousarray(np.r_[tgt, outl])
    ref = orc.expectation_step(src, tgt, 0.01, 0.15)
    orefs = {k: orc.registration(src, tgt, k[0], w=0.1, maxiter=6, tol=-1.0, update_scale=k[1])[0]
             for k in (("rigid", True), ("affine", True), ("rigid", False))}

    def body(comm):
        r = cpd.RigidCPD(src, comm=comm)
        es = r.expectation_step(src, tgt, 0.01, 0.15)
        lo, hi = comm.shard_bounds(tgt.shape[0])
        np.testing.assert_allclose(es.pt1, ref.pt1[lo:hi], rtol=2e-5, atol=1e-12)       # pt1: the local shard
        np.testing.assert_allclose(es.p1, ref.p1, rtol=2e-5, atol=1e-9)                 # p1 / px / n_p: global sums
        np.testing.assert_allclose(es.px, ref.px, rtol=2e-5, atol=2e-5 * np.abs(ref.px).max())
        assert es.n_p == pytest.approx(ref.n_p, rel=1e-6)
        out = [es.p1.tobytes()]
        for (kind, us), oref in orefs.items():
            kw = {} if kind == "affine" else {"update_scale": us}
            res = cpd.registration_cpd(src, tgt, kind, w=0.1, maxiter=6, tol=-1.0, comm=comm, **kw)
            lin = res.transformation.rot if kind == "rigid" else res.transformation.b
            np.testing.assert_allclose(lin, oref.params[0], atol=1e-5)
            np.testing.assert_allclose(res.transformation.t, oref.params[1], atol=1e-5)
            assert res.sigma2 == pytest.approx(oref.sigma2, rel=1e-6)
            out.append((res.sigma2, lin.tobytes()))
        m = r.maximization_step(tgt, es)                                                # M-step from a sharded EstepResult
        np.testing.assert_allclose(m.transformation.rot, orc.mstep_rigid(src, tgt, ref).params[0], atol=1e-5)
        return out

    results = _run_ranks(world, body)
    assert all(r == results[0] for r in results), "ranks disagree"


def test_sharded_nonrigid_dense_lowrank_constrained(emulated, monkeypatch):
    monkeypatch.setenv("CPD_EMU_DEVICES", "2")
    src, _ = orc.synthetic_pair(260)
    f = np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.7], [0.3, 0.0, 1.0]])
    tgt = src + 0.03 * np.sin(2 * np.pi * src.dot(f)) + 0.002 * np.random.default_rng(9).standard_normal(src.shape)
    tgt = np.ascontiguousarray(tgt[np.random.default_rng(1).permutation(260)][:251])
    dense_ref, _ = orc.registration(src, tgt, "nonrigid", maxiter=4, tol=-1.0, beta=1.0, lmd=1.5, w=0.05)
    g = orc.rbf_kernel_f32(src, src, 1.0)
    idx_s, idx_t = np.arange(0, 250, 10), np.arange(0, 250, 10)
    cons_ref, _ = orc.registration(src, tgt, "nonrigid_constrained", maxiter=3, tol=-1.0, beta=1.0, lmd=1.5, alpha=1e-2,
                                   idx_source=idx_s, idx_target=idx_t)

    def body(comm):
        a = cpd.NonRigidCPD(src, beta=1.0, lmd=1.5, comm=comm)
        ra = a.registration(tgt, w=0.05, maxiter=4, tol=-1.0)
        assert ra.sigma2 == pytest.approx(dense_ref.sigma2, rel=1e-5)
        np.testing.assert_allclose(a.moved_source(), src + g.dot(dense_ref.params[0]), atol=2e-5)
        b = cpd.NonRigidCPD(src, beta=1.0, lmd=1.5, comm=comm, low_rank=40)
        rb = b.registration(tgt, w=0.05, maxiter=4, tol=-1.0)
        assert rb.sigma2 == pytest.approx(dense_ref.sigma2, rel=1e-4)
        c = cpd.ConstrainedNonRigidCPD(src, beta=1.0, lmd=1.5, alpha=1e-2, idx_source=idx_s, idx_target=idx_t, comm=comm)
        rc = c.registration(tgt, maxiter=3, tol=-1.0)
        assert rc.sigma2 == pytest.approx(cons_ref.sigma2, rel=1e-5)
        return (ra.sigma2, rb.sigma2, rc.sigma2, a.moved_source().tobytes(), rb.transformation.w.tobytes())

    results = _run_ranks(2, body)
    assert results[0] == results[1], "ranks disagree"


def test_sharded_range_finder_gives_the_single_rank_factors(emulated, monkeypatch):
    """The G X products are split over the ranks' row shares and gathered by an all-reduce of value + zeros: the factors must be
    bit-identical to the single-rank ones."""
    monkeypatch.setenv("CPD_EMU_DEVICES", "3")
    src, tgt = orc.synthetic_pair(333)
    single = cpd.NonRigidCPD(src, beta=1.5, low_rank=30)
    single.registration(tgt, maxiter=1, tol=-1.0)
    q1, b1 = single._nr_factors

    def body(comm):
        reg = cpd.NonRigidCPD(src, beta=1.5, low_rank=30, comm=comm)
        reg.registration(tgt, maxiter=1, tol=-1.0)
        return reg._nr_factors[0].tobytes(), reg._nr_factors[1].tobytes()

    for q, b in _run_ranks(3, body):
        assert q == q1.tobytes() and b == b1.tobytes()
