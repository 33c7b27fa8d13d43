"""Ownership of the library's device memory, pinned memory and events, observed on the CPU emulation (tests/emu).

A copy of the emulated library is linked with a ledger (tests/emu_ledger.cpp) in front of its allocation and event stand-ins
(cpd_emu_alloc_stats).  Each scenario runs through the C ABI, closes every handle, and must leave the ledger where it found it:
no block, byte or event left behind, and no free of a pointer the runtime never handed out.  A second step at unchanged sizes
must allocate nothing, because cudaMalloc and cudaFree synchronise the device.
"""
import ctypes
import gc
import hashlib
import os
import subprocess

import numpy as np
import pytest

from probreg_b200 import _cabi
from probreg_b200 import gauss_transform as gt

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LEDGER_SRC = os.path.join(HERE, "emu_ledger.cpp")
WRAPPED = ("cudaMalloc", "cudaFree", "cudaMallocHost", "cudaFreeHost", "cudaEventCreate", "cudaEventDestroy")


@pytest.fixture(scope="module")
def ledger_lib_path(emu_lib_path):
    """The emulated library of tests/emu/build.py (its generated source), linked with the ledger."""
    build = os.path.dirname(emu_lib_path)
    emu = os.path.join(ROOT, "tests", "emu")
    gen, runtime = os.path.join(build, "cpd_b200_emu.cpp"), os.path.join(emu, "emu_runtime.cpp")
    out, obj = os.path.join(build, "libcpd_b200_emu_ledger.so"), os.path.join(build, "emu_runtime_base.o")
    stamp = os.path.join(build, "ledger_stamp")
    h = hashlib.sha256()
    for f in (os.path.join(build, "stamp"), runtime, os.path.join(emu, "cuda_runtime.h"), LEDGER_SRC, __file__):
        with open(f, "rb") as fh:
            h.update(fh.read())
    if os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return out
    flags = ["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-I" + emu, "-I" + build,
             "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "probreg_b200", "csrc")]
    subprocess.check_call(flags + ["-c", "-o", obj, runtime] + ["-D%s=emu_base_%s" % (f, f) for f in WRAPPED])
    subprocess.check_call(flags + ["-shared", "-o", out, gen, obj, LEDGER_SRC, "-ldl", "-lpthread"])
    with open(stamp, "w") as fh:
        fh.write(h.hexdigest())
    return out


@pytest.fixture
def emulated(ledger_lib_path):
    """The ledger's library in place of the loaded one for the duration of one test (as conftest's `emulated`)."""
    saved = _cabi._lib
    _cabi._lib = _cabi._load(ledger_lib_path)
    try:
        yield _cabi._lib
    finally:
        _cabi._lib = saved


KEYS = ("dev_blocks", "dev_bytes", "dev_allocs", "pin_blocks", "pin_bytes", "pin_allocs", "unknown_frees", "ev_created",
        "ev_destroyed")


def ledger(lib):
    out = (ctypes.c_longlong * len(KEYS))()
    lib.cpd_emu_alloc_stats(out)
    return dict(zip(KEYS, out))


def alloc_calls(lib, fn):
    """allocation calls (device and pinned) made by fn()"""
    a = ledger(lib)
    fn()
    b = ledger(lib)
    return (b["dev_allocs"] - a["dev_allocs"]) + (b["pin_allocs"] - a["pin_allocs"])


def assert_balanced(lib, before):
    gc.collect()
    after = ledger(lib)
    for k in ("dev_blocks", "dev_bytes", "pin_blocks", "pin_bytes", "unknown_frees"):
        assert after[k] == before[k], (k, before, after)
    assert after["ev_created"] - before["ev_created"] == after["ev_destroyed"] - before["ev_destroyed"], (before, after)


def clouds(m, n, dim=3, seed=0):
    rng = np.random.default_rng(seed)
    src = rng.random((m, dim))
    rot = np.eye(dim)
    rot[:2, :2] = [[np.cos(0.2), -np.sin(0.2)], [np.sin(0.2), np.cos(0.2)]]
    tgt = src[rng.permutation(m)[:n]] @ rot.T + 0.05
    return src, tgt


def handle(src, tgt):
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(tgt)
    return h


def sc_create_destroy(lib):
    for dim in (2, 3):
        _cabi.Handle(dim).close()


def sc_em_run(lib):
    for kind in (_cabi.TF_RIGID, _cabi.TF_AFFINE):
        src, tgt = clouds(160, 150)
        h = handle(src, tgt)
        h.set_state(kind, True, 0.1, np.eye(3), np.zeros(3), 1.0, h.sigma2_init(), 0.0)
        h.em_run(3, -1.0)
        assert alloc_calls(lib, lambda: h.em_step()) == 0
        h.close()


def sc_estep_mstep(lib):
    src, tgt = clouds(170, 140)
    h = handle(src, tgt)
    pt1, p1, px, n_p = h.estep(src, 0.05, 0.1)
    h.mstep(_cabi.TF_RIGID, True, pt1, p1, px, n_p)
    h.bcpd_estep(src, 1.0, np.full(170, 1.0 / 170), np.ones(170), 0.05, 0.1)
    h.estep(src, 1e-4, 0.0)
    h.close()


def sc_nonrigid(lib):
    src, tgt = clouds(150, 140)
    s2 = 0.05
    h = handle(src, tgt)
    h.nonrigid_begin(2.0, 2.0, s2, 0.0)
    h.nonrigid_step()
    assert alloc_calls(lib, h.nonrigid_step) == 0
    h.nonrigid_w()
    h.nonrigid_lowrank_begin(2.0, 2.0, s2, 0.0, 20)
    h.nonrigid_step()
    assert alloc_calls(lib, h.nonrigid_step) == 0
    h.nonrigid_w()
    h.nonrigid_lowrank_factors()
    h.nonrigid_restart(2.0, s2, 0.1)
    h.nonrigid_step()
    idx = np.arange(0, 150, 10)
    p1t = np.zeros(150)
    p1t[idx] = 1.0
    pxt = np.zeros((150, 3))
    pxt[idx] = src[idx] + 0.05
    h.nonrigid_set_prior(1e-2, p1t, pxt)
    h.nonrigid_step()
    pt1, p1, px, _ = h.estep(src, s2, 0.0)
    h.nonrigid_mstep(pt1, p1, px, s2)
    h.nonrigid_begin(2.0, 2.0, s2, 0.0)              # back to the dense G on the same handle
    h.nonrigid_step()
    h.close()


def sc_bcpd(lib):
    src, tgt = clouds(140, 130)
    h = handle(src, tgt)
    h.bcpd_begin(np.eye(140, dtype=np.float32), 2.0, 1e20, 0.1, 0.0)
    h.bcpd_step()
    assert alloc_calls(lib, h.bcpd_step) == 0
    h.bcpd_get(v=True, moved=True, alpha=True, sigma_diag=True)
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    h.bcpd_step()
    assert alloc_calls(lib, h.bcpd_step) == 0
    h.bcpd_lowrank_factors()
    h.bcpd_get(v=True, moved=True)
    h.close()
    # low-rank BCPD begun on a handle with a live non-rigid loop
    h = handle(src, tgt)
    h.nonrigid_lowrank_begin(2.0, 2.0, 0.05, 0.0, 20)
    h.nonrigid_step()
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 0.1, 0.0, 20)
    h.bcpd_step()
    h.close()


def sc_gmmtree(lib):
    src, tgt = clouds(200, 180)
    h = handle(src, tgt)
    h.gmmtree_build(1, 1e-3, 1e-3, np.arange(0, 200, 25), maxiter=5)
    h.gmmtree_assign()
    pi, mu, cov = h.gmmtree_nodes()
    h.gmmtree_estep(np.eye(3), np.zeros(3), 0.01)
    assert alloc_calls(lib, lambda: h.gmmtree_estep(np.eye(3), np.zeros(3), 0.01)) == 0
    h.gmmtree_load(1, pi, mu, cov)
    h.gmmtree_estep(np.eye(3), np.zeros(3), 0.01)
    h.close()


def sc_features(lib):
    src, tgt = clouds(120, 100)
    h = handle(src, tgt)
    h.gmm_fit(4, [0, 30, 60, 90], max_iter=5)
    h.close()
    _cabi.l2_dist(src[:20], np.full(20, 0.05), tgt[:15], np.full(15, 1.0 / 15), 0.5)
    _cabi.ocsvm_fit(src[:60], 0.2, 2.0)


def sc_filterreg(lib):
    src, tgt = clouds(150, 130)
    loop = _cabi.FilterRegLoop(src, tgt, update_sigma2=True)
    loop.step(np.eye(3), np.zeros(3), 0.01, 0.0)
    assert alloc_calls(lib, lambda: loop.step(np.eye(3), np.zeros(3), 0.01, 0.0)) == 0
    loop.last_estep()
    loop.stage_ms()
    del loop
    _cabi.filterreg_estep(src, tgt, 0.01, True, target_normals=np.tile([0.0, 0.0, 1.0], (130, 1)))
    f = np.random.default_rng(1).random((90, 3)).astype(np.float32) * 4
    _cabi.lattice_filter(f, np.ones((90, 2), np.float32))
    _cabi.lattice_filter(f, None, with_blur=False)


def sc_gauss_transform(lib):
    src, tgt = clouds(100, 80)
    gt.GaussTransform(src, 0.3).compute(tgt)
    gt.GaussTransform(src, 0.3).compute(tgt, np.ones((2, 100)))


def sc_alternating_sizes(lib):
    h = _cabi.Handle(3)
    for k in range(3):
        for m, n in ((120, 90), (260, 300)):
            src, tgt = clouds(m, n, seed=k)
            h.set_source(src)
            h.set_target(tgt)
            h.estep(src, 0.05, 0.1)
    h.close()


def sc_argument_errors(lib):
    err = _cabi.CpdError
    p = ctypes.c_void_p()
    assert lib.cpd_create(ctypes.byref(p), 0, 4, None) != 0
    src, tgt = clouds(100, 90)
    h = handle(src, tgt)
    bad = np.full((100, 3), np.nan)
    calls = [
        lambda: lib.cpd_set_source(h._h, _cabi.dptr(src), 0),
        lambda: h.set_target(tgt, n_global=10),
        lambda: h.set_state(7, True, 0.1, np.eye(3), np.zeros(3), 1.0, 0.1, 0.0),
        lambda: h.estep(src, -1.0, 0.1),
        lambda: h.bcpd_estep(src, 1.0, np.zeros(100), np.ones(100), 0.05, 0.1),
        lambda: h.mstep(7, True, np.ones(90), np.ones(100), src, 1.0),
        lambda: h.nonrigid_begin(-1.0, 2.0, 0.1, 0.0),
        lambda: h.nonrigid_lowrank_begin(2.0, 2.0, 0.1, 0.0, 0),
        lambda: h.nonrigid_step(),
        lambda: h.bcpd_begin(np.eye(100, dtype=np.float32), -2.0, 1e20, 0.1, 0.0),
        lambda: lib.cpd_bcpd_lowrank_begin(h._h, 1.0, 2.0, 1e20, 0.1, 0.0, 0, 2, 0),
        lambda: h.bcpd_step(),
        lambda: h.gmmtree_build(1, 1e-3, 1e-3, np.full(8, 1000)),
        lambda: h.gmmtree_estep(np.eye(3), np.zeros(3), 0.01),
        lambda: h.gmm_fit(4, [0, 0, 1, 2]),
        lambda: _cabi.l2_dist(src, np.ones(100), tgt, np.ones(90), -1.0),
        lambda: _cabi.ocsvm_fit(src, 2.0, 1.0),
        lambda: _cabi.filterreg_estep(bad, tgt, 0.01, False),
        lambda: _cabi.FilterRegLoop(src, tgt, alpha=np.inf),
        lambda: _cabi.lattice_filter(np.full((10, 3), 1e9, np.float32), np.ones((10, 1), np.float32)),
        lambda: gt.GaussTransform(src, -1.0).compute(tgt),
    ]
    for k, call in enumerate(calls):
        try:
            r = call()
        except (err, ValueError):
            continue
        assert isinstance(r, int) and r != 0, k
    loop = _cabi.FilterRegLoop(src, tgt)
    with pytest.raises(err):
        loop.step(np.eye(3), np.zeros(3), -1.0, 0.0)
    del loop
    h.close()


SCENARIOS = [sc_create_destroy, sc_em_run, sc_estep_mstep, sc_nonrigid, sc_bcpd, sc_gmmtree, sc_features, sc_filterreg,
             sc_gauss_transform, sc_alternating_sizes, sc_argument_errors]


@pytest.mark.parametrize("scenario", SCENARIOS, ids=[s.__name__[3:] for s in SCENARIOS])
def test_scenario_returns_every_block_and_event(emulated, scenario):
    gc.collect()
    before = ledger(emulated)
    scenario(emulated)
    assert_balanced(emulated, before)
