"""CPU evidence for the precision design: the arithmetic the CUDA kernels perform -- FP32 pair maths
with the same FMA chains, integer offsets, two-level FP32 group sums, FP64 beyond, residual-form M-step -- emulated in
numpy (tools/emulate_resid.py, exactly rounded exp2 instead of MUFU.EX2) meets the north-star tolerances against the
fixtures produced by the reference.  The GPU tests check the real kernels; this one runs without a GPU."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "tools"))
import emulate_resid as er  # noqa: E402


def test_emulated_kernel_arithmetic_meets_the_bar_on_the_bunny(bunny):
    with np.errstate(over="ignore"):
        order_s, order_t = er.morton_order(bunny["source"]), er.morton_order(bunny["target"])
        s2 = er.registration(bunny["source"][order_s], bunny["target"][order_t], 10)
    ref = float(bunny["rigid10_sigma2"])
    assert abs(s2 - ref) <= 1e-6 * ref, (s2, ref)


def test_flat_fp32_sums_would_not(bunny):
    """The failure mode the design avoids: one FP32 accumulator per 128 terms, caller's (unsorted) order."""
    g = load_golden("synthetic1500.npz")
    with np.errstate(over="ignore"):
        s2 = er.registration(g["source"][:600], g["target"][:600], 12, sub=128, grp=0)
        s2_good = er.registration(g["source"][:600], g["target"][:600], 12, acc64=True)
    assert abs(s2 - s2_good) > 3e-7 * s2_good          # measurably worse than exact accumulation ...
    with np.errstate(over="ignore"):
        o_s, o_t = er.morton_order(g["source"][:600]), er.morton_order(g["target"][:600])
        s2_design = er.registration(g["source"][:600][o_s], g["target"][:600][o_t], 12)
    assert abs(s2_design - s2_good) < 1.5e-7 * s2_good  # ... while Z-order + group sums stay close to it
