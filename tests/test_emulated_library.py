"""The GPU parity tests, executed on the CPU against the emulated library (tests/emu).

What this buys: the container the CPU suite runs in has no GPU, so without this nothing under
probreg_b200/csrc would be executed before the round-end GPU run.  The emulation compiles the SAME sources
(cpd_b200.cu with its launches rewritten, kernels.cuh with host stand-ins for the inline PTX) and runs blocks,
warps, barriers, shuffles, the TMA/mbarrier ring and the launch sequence for real -- so index arithmetic, buffer
sizes, work lists, permutations, reductions, the M-step algebra and the C-ABI plumbing are all exercised.
What it does not model: timing, MUFU.EX2's approximation error, memory-ordering races, real cuSOLVER/NCCL.
The test bodies are the GPU tests' own (imported), at sizes the fibers finish in seconds.
"""
import numpy as np
import pytest

import test_cuda_edges as E
import test_cuda_parity as P

CASES = [
    (P.test_squared_kernel_sum_known_answer, {}),
    (P.test_rbf_kernel_symmetric_and_matches_reference, {}),
    (P.test_sigma2_init, {"bunny": "fixture"}),
    (P.test_estep_bunny_vs_reference, {"bunny": "fixture", "tag": "e0", "w": 0.0}),
    (P.test_estep_bunny_vs_reference, {"bunny": "fixture", "tag": "e0w", "w": 0.3}),
    (P.test_estep_outliers_vs_reference, {"syn1500": "fixture", "tag": "dead"}),
    (P.test_estep_outliers_vs_reference, {"syn1500": "fixture", "tag": "deadw"}),
    (P.test_estep_ragged_sizes, {"m": 1, "n": 1, "dim": 3, "w": 0.0}),
    (P.test_estep_ragged_sizes, {"m": 1, "n": 700, "dim": 3, "w": 0.2}),
    (P.test_estep_ragged_sizes, {"m": 700, "n": 1, "dim": 3, "w": 0.0}),
    (P.test_estep_ragged_sizes, {"m": 1023, "n": 1025, "dim": 3, "w": 0.2}),
    (P.test_estep_ragged_sizes, {"m": 1025, "n": 511, "dim": 3, "w": 0.0}),
    (P.test_estep_ragged_sizes, {"m": 91, "n": 91, "dim": 2, "w": 0.0}),
    (P.test_estep_ragged_sizes, {"m": 1500, "n": 333, "dim": 2, "w": 0.2}),
    (P.test_mstep_from_oracle_estep, {"kind": "rigid"}),
    (P.test_mstep_from_oracle_estep, {"kind": "rigid_noscale"}),
    (P.test_mstep_from_oracle_estep, {"kind": "affine"}),
    (P.test_mstep_2d_and_reflection, {}),
] + [
    (P.test_registration_vs_reference, dict(zip("fname,tag,tf_type,iters,w,kw,sk,tk".split(","), c), callbacks=(i % 2 == 0)))
    for i, c in enumerate(P.CASES)
] + [
    (P.test_estep_outliers_vs_reference, {"syn1500": "fixture", "tag": "mid"}),
    (P.test_estep_ragged_sizes, {"m": 2049, "n": 4097, "dim": 3, "w": 0.2}),
    (P.test_default_tolerance_stops_where_the_reference_does, {"bunny": "fixture", "tag": "rigid_default", "tf_type": "rigid"}),
    (P.test_default_tolerance_stops_where_the_reference_does, {"bunny": "fixture", "tag": "affine_default", "tf_type": "affine"}),
    (P.test_nonrigid_device_loop_2000_vs_oracle, {}),
    (P.test_estep_sigma_sweep_20k, {"s2": 1e-4}),                  # 20 tiles x 40 stages, culling instantiations, vs the C oracle
    (P.test_tf_init_params_and_reference_test_recipe, {}),
    (P.test_nonrigid_vs_reference, {"nonrigid_golden": "fixture"}),
    (P.test_constrained_nonrigid_vs_reference, {"nonrigid_golden": "fixture"}),
    (E.test_duplicate_points_and_exact_coincidence, {}),
    (E.test_identical_clouds_hit_the_sigma2_floor_like_the_reference, {}),
    (E.test_all_points_equal_and_collinear_clouds, {}),
    (E.test_extreme_sigma2, {"s2": 1e3}),
    (E.test_extreme_sigma2, {"s2": 1e-9}),
    (E.test_handle_reuse_with_other_sizes_and_families, {}),
    (E.test_inputs_are_not_modified_and_any_layout_is_accepted, {}),
    (E.test_same_sizes_new_data_on_one_handle_and_buffers_free_on_return, {}),
    (E.test_argument_errors, {}),
    (E.test_results_are_deterministic, {}),
    (E.test_gauss_transform_vs_direct, {}),
]


def _id(case):
    fn, kw = case
    return fn.__name__[5:] + "".join("-%s" % v for k, v in kw.items() if v != "fixture" and not isinstance(v, dict))


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_gpu_test_body_under_emulation(emulated, request, case):
    fn, kw = case
    args = {k: (request.getfixturevalue(k) if isinstance(v, str) and v == "fixture" else v) for k, v in kw.items()}
    fn(**args)


def test_culling_is_bit_exact_under_emulation(emulated, monkeypatch):
    """The exact-culling instantiations (two-level boxes) against the dense ones, bit for bit, at sizes fibers can do."""
    from oracle import cpd_oracle as orc
    from probreg_b200 import _cabi

    src, tgt = orc.synthetic_pair(6000)
    ts = orc.apply_rigid(src, orc.rot_z(30.0), np.array([0.1, -0.2, 0.3]))

    def run(no_cull):
        monkeypatch.setenv("CPD_B200_NO_CULL", "1" if no_cull else "0")
        h = _cabi.Handle(3)
        h.set_source(ts)
        h.set_target(tgt)
        return [h.estep(ts, s2, 0.1) for s2 in (1e-5, 1e-4)]

    for a, b in zip(run(False), run(True)):
        for x, y in zip(a[:3], b[:3]):
            assert np.array_equal(x, y)
        assert a[3] == b[3]


@pytest.mark.parametrize("sms", [1, 3])
def test_multi_wave_work_lists_under_emulation(emulated, monkeypatch, sms):
    """Few resident CTA slots -> several waves and other stage splits per tile; results must not depend on that."""
    from oracle import cpd_oracle as orc
    from probreg_b200 import cpd

    monkeypatch.setenv("CPD_EMU_SMS", str(sms))
    rng = np.random.default_rng(sms)
    src, tgt = rng.random((2500, 3)), rng.random((1800, 3)) + 0.02
    es = cpd.RigidCPD(src).expectation_step(src, tgt, 0.004, 0.1)
    ref = orc.expectation_step(src, tgt, 0.004, 0.1)
    np.testing.assert_allclose(es.pt1, ref.pt1, rtol=2e-5)
    np.testing.assert_allclose(es.p1, ref.p1, rtol=2e-5, atol=1e-9)
    np.testing.assert_allclose(es.px, ref.px, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("unit,last_cost", [("stage", "1.0"), ("subchunk", "1.0"), ("subchunk", "0.3"), ("stage", "0.6")])
def test_pass1_plan_switches_under_emulation(emulated, monkeypatch, unit, last_cost):
    """Pass 1's work plan (tuning switches): whole stages or sub-chunks as the unit of the cuts, any cost of the
    last tile -- items that begin and end inside a TMA stage, a last tile whose warps of padding leave the kernel at once (1300
    targets: 276 in the second tile, 3 of its 8 warps alive).  The plan must never show in the results."""
    from oracle import cpd_oracle as orc
    from probreg_b200 import cpd

    monkeypatch.setenv("CPD_B200_PLAN_UNIT", unit)
    monkeypatch.setenv("CPD_B200_PLAN_LAST_COST", last_cost)
    monkeypatch.setenv("CPD_EMU_SMS", "4")
    rng = np.random.default_rng(5)
    src, tgt = rng.random((2300, 3)), rng.random((1300, 3)) + 0.02
    es = cpd.RigidCPD(src).expectation_step(src, tgt, 0.004, 0.1)
    ref = orc.expectation_step(src, tgt, 0.004, 0.1)
    np.testing.assert_allclose(es.pt1, ref.pt1, rtol=2e-5)
    np.testing.assert_allclose(es.p1, ref.p1, rtol=2e-5, atol=1e-9)
    np.testing.assert_allclose(es.px, ref.px, rtol=2e-5, atol=2e-5)


def test_results_do_not_depend_on_the_thread_schedule(emu_lib_path):
    """Same inputs under three fiber schedules (in order, reversed, a random permutation per round): bit-identical results."""
    import os
    import subprocess
    import sys

    probe = os.path.join(os.path.dirname(emu_lib_path), "..", "sched_probe.py")
    digests = []
    for mode in ("rr", "reverse", "random:11"):
        env = dict(os.environ, CPD_EMU_SCHED=mode)
        r = subprocess.run([sys.executable, probe, emu_lib_path], capture_output=True, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        digests.append(r.stdout.strip().splitlines()[-1])
    assert digests[0] == digests[1] == digests[2], digests


def test_parity_survives_a_mufu_like_ex2(emu_lib_path):
    """Re-run a slice of the emulated tests with ex2 perturbed by up to 2^-22 relative, smoothly in the fractional part of its
    argument (CPD_EMU_EX2=mufu): parity must not hinge on an exact exp2 -- the two passes see identical arguments, so the error
    cancels in K / sum K."""
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, CPD_EMU_EX2="mufu")
    sel = "estep_bunny or registration_vs_reference or default_tolerance or bcpd_estep_vs_reference or lowrank_vs_oracles"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "not gpu", "-p", "no:cacheprovider", "-k", sel,
                        os.path.join(here, "test_emulated_library.py"), os.path.join(here, "test_zz_bcpd.py"),
                        os.path.join(here, "test_zz_lowrank.py")], capture_output=True, text=True, env=env, timeout=1500, cwd=here)
    assert r.returncode == 0, r.stdout[-3000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


def test_emulation_is_not_reachable_from_the_package(emu_lib_path):
    """The package loads probreg_b200/libcpd_b200.so (or another build of it named by CPD_B200_LIB) and nothing else; pointing
    CPD_B200_LIB at the emulation is refused (a subprocess, so that this process's loaded library is untouched)."""
    import os
    import subprocess
    import sys

    from probreg_b200 import _cabi

    assert os.path.basename(_cabi.LIB_PATH) == "libcpd_b200.so" or "CPD_B200_LIB" in os.environ
    assert os.sep + "tests" + os.sep in emu_lib_path
    pkg = os.path.dirname(_cabi.__file__)
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            text = open(os.path.join(pkg, f)).read()
            assert "tests/emu" not in text and "_emu." not in text and "emu_" not in text, f       # no path to the emulation build
    env = dict(os.environ, CPD_B200_LIB=emu_lib_path)
    code = ("from probreg_b200 import _cabi\n"
            "try:\n    _cabi.lib()\n    print('LOADED')\n"
            "except _cabi.CpdError as e:\n    print('REFUSED', 'emulation' in str(e))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=120,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.stdout.strip() == "REFUSED True", r.stdout + r.stderr
