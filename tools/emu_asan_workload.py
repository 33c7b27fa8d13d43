"""AddressSanitizer sweep of the emulated library (test infrastructure; see tests/emu/README.md).

Build:  g++ -O1 -g -std=c++17 -fPIC -shared -ffp-contract=off -fno-strict-aliasing -w -fsanitize=address -fno-omit-frame-pointer -DEMU_UCONTEXT \
        -Itests/emu -Itests/emu/_build -Iinclude -Iprobreg_b200/csrc -o tests/emu/_build/libcpd_b200_emu_asan.so \
        tests/emu/_build/cpd_b200_emu.cpp tests/emu/emu_runtime.cpp -ldl        (after python tests/emu/build.py)
Run:    ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 LD_PRELOAD=$(gcc -print-file-name=libasan.so) \
        python tools/emu_asan_workload.py
"""
import sys
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from probreg_b200 import _cabi
_cabi.LIB_PATH = os.path.join(ROOT, 'tests', 'emu', '_build', 'libcpd_b200_emu_asan.so')
from probreg_b200 import cpd, bcpd, gauss_transform as gt
from oracle import cpd_oracle as orc
rng = np.random.default_rng(0)
for (m, n) in [(1, 1), (700, 1), (1, 700), (1023, 1025), (1500, 333)]:
    src, tgt = rng.random((m, 3)), rng.random((n, 3))
    cpd.RigidCPD(src).expectation_step(src, tgt, 0.01, 0.1)
print("estep ok")
src, tgt = orc.synthetic_pair(1300)
cpd.registration_cpd(src, tgt, maxiter=3, tol=-1)
cpd.registration_cpd(src, tgt, "affine", maxiter=3, tol=-1)
ts = orc.apply_rigid(src, orc.rot_z(30.0), np.array([0.1, -0.2, 0.3]))
h = _cabi.Handle(3); h.set_source(ts); h.set_target(tgt); h.estep(ts, 1e-5, 0.1); h.estep(ts, 1e-4, 0.0)
print("reg + cull ok")
s2, t2 = rng.random((200, 2)), rng.random((150, 2))
cpd.registration_cpd(s2, t2, maxiter=2, tol=-1)
a = cpd.NonRigidCPD(src[:300], low_rank=40); a.registration(tgt[:310], maxiter=2, tol=-1); a.moved_source()
b = cpd.NonRigidCPD(src[:300]); b.registration(tgt[:310], maxiter=2, tol=-1)
idx = np.arange(0, 300, 10)
c = cpd.ConstrainedNonRigidCPD(src[:300], idx_source=idx, idx_target=idx, alpha=1e-2, low_rank=30); c.registration(tgt[:310], maxiter=2, tol=-1)
es_ = orc.expectation_step(src[:300], tgt[:310], 0.01, 0.05)
b.maximization_step(tgt[:310], cpd.EstepResult(*es_), 0.01); a.maximization_step(tgt[:310], cpd.EstepResult(*es_), 0.01)
c.maximization_step(tgt[:310], cpd.EstepResult(*es_), 0.01)
a.registration(tgt[:290] + 0.01, maxiter=2, tol=-1)            # restart path: factors kept
d = cpd.NonRigidCPD(src[:120], low_rank=120); d.registration(tgt[:100], maxiter=1, tol=-1)   # rank == M
print("nonrigid ok")
bcpd.CombinedBCPD(src[:257]).expectation_step(src[:257], tgt[:513], 1.0, 1.0 / 257, np.ones(257), 0.02, 0.1)
gt.GaussTransform(src[:300], 0.3).compute(tgt[:100], rng.standard_normal((5, 300)))
r = cpd.RigidCPD(src); es = r.expectation_step(src, tgt, 0.02, 0.0); r.maximization_step(tgt, es)
print("all ok")
