"""The CPD E-step element-wise at the benchmark's sizes, against the exact sparse float64 reference (oracle/sparse_oracle.py)
evaluated on the kernels' own FP32 inputs.

Every case calls ``_cabi.Handle`` with an explicit ``frame_origin``, so ``pack_kernel``'s coordinates a_m = fl32(sk (ts_m - c_x)),
b_n = fl32(sk (x_n - c_x)) are known bit for bit and the reference computes K = 2^-u, u = |a_m - b_n|^2, in float64 from them.
Each case runs twice, with the culling instantiations and with ``CPD_B200_NO_CULL=1``, and checks
  (a) the pt1 == 0 pattern equals the reference's (columns whose nearest exponent lies in float64's denormal band excluded);
  (b) |got - ref| <= bound element-wise for pt1, p1 and px (the bound below);
  (c) n_p and sum px against the conservation laws (1e-7 / 1e-6, as the other full-size tests);
  (d) culled and unculled outputs bit-identical.

The bound.  eps = 2^-24 (FP32 rounding), eta = 2^-22 (MUFU.EX2 relative error), log2 units for exponents.

1. One pair (pass1_sum / pass2_kernel): dx = fl(a_x - b_x) (relative eps each, so the squares move by 2 eps u in all), then
   t' = fl(dz^2 + fl(dy^2 + fl(dx^2 - o_n))) -- three FMAs, each rounding at most eps of its result, whose magnitude is at most
   u + o_n.  Pass 1 seeds o_n from 128 sources of the nearest source stage and lowers it only when a sub-chunk sum reaches
   2^100, so o_n <= u_min,n + 101 (the floor included).  Hence |t' - (u - o)| <= delta_mn = eps (2u + 3 (u + u_min,n + 101)).
   The weighted E-step (WGT) adds la'_m with a fourth rounding (|t' + la| <= u + la + o) and may hold la'_m one float32 ulp
   (2 eps la') away from the reference (bcpd_la_kernel's FP64 log2 is not numpy's): delta_mn = eps (2u + 4 (2 (u + la) + 101)
   + 2 la).  The pair's K is then off by ln2 delta_mn + eta relative.
2. Column sum (pass 1, finalize1): FP32 groups of 8 from zero, 8 group sums joined, FP64 beyond: 14 eps of the sum; terms
   flushed below 2^-126 (ex2.approx.ftz): < 2^-125 of the column's largest each.  Relative error of sum K:
   r_n = ln2 dbar_n + eta + 15 eps + 2^-125 cnt_n, dbar_n the K-weighted mean of delta over the column.
   pt1 = S / (S + c) moves by pt1 (1 - pt1) r_n (exactly 1.0 when w = 0), plus 2^-52 (cnt_n + 4) pt1 for finalize1's FP64
   log2 / exp2 and the reference's own float64 sum over the column.
3. P_mn = 2^(o - u) rn_n (pass 2, the same offset): rn rounded to float32 (eps) and the product (eps); the row sum p1_m in
   FP32 groups (14 eps).  |dp1_m| <= ln2 sum_n P_mn (delta_mn + dbar_n) + (2 eta + 32 eps) p1_m + 2^-125 (cnt_m + 1):
   the last term is the P_mn under FP32's range that pass 2 loses -- where w > 0 and a column is weak, rn_n = 2^-o / den_n
   itself falls below 2^-126 -- each below 2^-125 of its column's largest P, and the pairs the reference cuts (< 2^-139 in all).
   Worse, pass 2's factor rn_n = 2^-o_n / den_n is a float32, and with the offset up to 101 above u_min,n it is only bounded
   below by 2^-101 Pmax_n (Pmax_n = 2^-u_min,n / den_n).  Where Pmax_n < 2^-25 (w > 0, a weak column), rn_n may be subnormal
   (an absolute 2^-149) or flush to 0, and P_mn = 2^(o - u) rn_n is off by up to 2^-(u_mn - u_min,n) min(Pmax_n, 2^-49):
   summed per row (``row_sub``; factor 1 with per-source exponents).  On the H100 at sigma2 = 1e-6, w = 0.1 a column with
   pt1 = 3e-22 lost its whole P this way (the offset had overshot by ~100): an absolute 2.9e-22, inside this term.
4. px_m = p1_m ts_m + sum_n P_mn (b_n - a_m) / sk (finalize2 + uncentre in FP64): |dpx_m| <= |dp1_m| (|ts_m| + d) + 16 eps p1_m d,
   d = the largest kept |a - b| / sk (the FP32 sums of P dx, and dx's own rounding).

The offset term (3 (u_min + 101) eps) dominates: the bound is ~1e-5 relative where u is small and ~1e-4 at sigma2 = 1e-6
(u ~ 200 for the synthetic pair's 0.01 noise); a 1-ulp error of the packed coordinates moves K by ~1e-3 there and a K off by
2^-12 relative in every other source row breaks it too (the two sharpness tests).  Offsets below the column's smallest u + 101
make the error smaller, never larger, so 2^-20 is inside what the kernels may legitimately differ by.

The E-step inside the registration loop (``cpd_em_step``) forms a_m from the centred sources, the device centroid and the
transform (FMA-contracted FP64) instead of an uploaded ts: a_m may differ from the reference's by one float32 ulp (2 eps |a_m|),
which moves u by up to 4 eps |a_m| sqrt(u) -- added to delta_mn for those cases.
"""
import os

import numpy as np
import pytest

from oracle import cpd_oracle as orc
from oracle import sparse_oracle as so
from probreg_b200 import _cabi

EPS, ETA, LN2 = 2.0 ** -24, 2.0 ** -22, np.log(2.0)
TRUE_T = np.array([0.1, -0.2, 0.3])
ROWS = []           # (case, instantiation, worst error / bound of pt1, p1, px): printed at the end of the module


def _delta_plain(u, la, col_umin):
    return EPS * (2.0 * u + 3.0 * (u + col_umin + 101.0))


def _delta_wgt(u, la, col_umin):
    return EPS * (2.0 * u + 4.0 * (2.0 * (u + la) + 101.0) + 2.0 * la)


def _delta_loop(anorm):
    def f(u, la, col_umin):
        return _delta_plain(u, la, col_umin) + 4.0 * EPS * anorm * np.sqrt(u)
    return f


def bounds(ref, ts):
    """Per-element bounds (pt1, p1, px) of section 1-4 of the module docstring from the sparse reference's sums."""
    es, ex = ref
    pt1 = es.pt1
    r = LN2 * ex.col_dbar + ETA + 15.0 * EPS + 2.0 ** -125 * ex.col_cnt
    b_pt1 = pt1 * (1.0 - pt1) * r + 2.0 ** -52 * (ex.col_cnt + 4) * pt1
    b_p1 = (LN2 * (ex.row_pd + ex.row_pdbar) + (2.0 * ETA + 32.0 * EPS) * es.p1 + 2.0 ** -125 * (ex.row_cnt + 1)
            + ex.row_sub)
    b_px = b_p1[:, None] * (np.abs(ts) + ex.dmax) + 16.0 * EPS * es.p1[:, None] * ex.dmax
    return b_pt1, b_p1, b_px


def worst(got, ref, bnd, live=None):
    err = np.abs(got - ref)
    if live is not None:
        err, bnd = err[live], bnd[live]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bnd > 0, err / bnd, np.where(err > 0, np.inf, 0.0))
    return float(q.max()) if q.size else 0.0


def handle_pair(dim, src, tgt, n_global, origin):
    """Two handles on the same clouds: culling instantiations allowed / CPD_B200_NO_CULL=1 (read at handle creation)."""
    out = []
    for no_cull in ("0", "1"):
        old = os.environ.get("CPD_B200_NO_CULL")
        os.environ["CPD_B200_NO_CULL"] = no_cull
        try:
            h = _cabi.Handle(dim)
        finally:
            if old is None:
                os.environ.pop("CPD_B200_NO_CULL")
            else:
                os.environ["CPD_B200_NO_CULL"] = old
        h.set_source(src)
        h.set_target(tgt, n_global=n_global, frame_origin=origin)
        out.append(h)
    return out


def check_outputs(name, outs, ref, ts, bcpd=False):
    """(a)-(d) of the module docstring for the (culled, unculled) outputs."""
    es, ex = ref
    b_pt1, b_p1, b_px = bounds(ref, ts)
    live = ~ex.band
    for inst, o in zip(("culled", "unculled"), outs):
        pt1, p1, px, n_p = o
        np.testing.assert_array_equal((pt1 == 0)[live], (es.pt1 == 0)[live], err_msg="%s %s: dead columns" % (name, inst))
        q = (worst(pt1, es.pt1, b_pt1, live), worst(p1, es.p1, b_p1), worst(px, es.px, b_px))
        ROWS.append((name, inst + (" weighted" if bcpd else ""), ex.pairs) + q)
        print("%-36s %-18s pairs %.2e  worst err/bound  pt1 %.3f  p1 %.3f  px %.3f" % ((name, inst + (" weighted" if bcpd else ""), ex.pairs) + q))
        assert max(q) <= 1.0, "%s %s: worst error / bound %s" % (name, inst, q)
        assert n_p == pytest.approx(p1.sum(), rel=1e-12)
        assert n_p == pytest.approx(pt1.sum(), rel=1e-7, abs=1e-300)
    for a, b in zip(outs[0], outs[1]):
        assert np.array_equal(a, b), "%s: culling changed a bit" % name


def run_case(name, src, tgt, ts, s2, w, n_global=None, origin=None, dim=3):
    origin = tgt.mean(0) if origin is None else origin
    hs = handle_pair(dim, src, tgt, n_global if n_global is not None else tgt.shape[0], origin)
    outs = [h.estep(ts, s2, w) for h in hs]
    for h in hs:
        h.close()
    ref = so.expectation_step(ts, tgt, s2, w, n_global=n_global, frame_origin=origin, pair_err=_delta_plain)
    check_outputs(name, outs, ref, ts)
    pt1, p1, px, n_p = outs[0]
    np.testing.assert_allclose(px.sum(0), (pt1[:, None] * tgt).sum(0), rtol=1e-6, atol=1e-300)      # (c)
    return outs[0], ref


# ---------------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------------
def pair(n, m=None, kind="rigid", dim=3):
    """The synthetic pair (sources at the transform of test_estep_sigma_sweep_20k, a half degree from the truth)."""
    m = n if m is None else m
    src, _ = orc.synthetic_pair(m, kind)
    _, tgt = orc.synthetic_pair(n, kind)
    if kind == "affine":
        lin = orc.rot_z(30.0).dot(np.diag([1.1, 0.9, 1.05]))
        lin[0, 1] += 0.05
        ts = orc.apply_affine(src, orc.rot_z(-0.5).dot(lin), TRUE_T)
    else:
        ts = orc.apply_rigid(src, orc.rot_z(29.5), TRUE_T)
    if dim == 2:
        src, tgt, ts = src[:, :2].copy(), tgt[:, :2].copy(), ts[:, :2].copy()
    return np.ascontiguousarray(src), np.ascontiguousarray(tgt), np.ascontiguousarray(ts)


def variant(src, tgt, ts, kind, seed=7):
    rng = np.random.default_rng(seed)
    if kind == "shift":                              # frame precision: the clouds 1e3 away from the origin of coordinates
        return src + 1e3, tgt + 1e3, ts + 1e3
    if kind == "grid":                               # exact duplicates and targets exactly on sources (u = 0, Morton ties)
        q = 2.0 ** -8
        ts = np.round(ts / q) * q
        ts[1::5] = ts[0::5][: len(ts[1::5])]
        tgt = np.round(tgt / q) * q
        idx = rng.choice(len(ts), len(tgt) // 4, replace=True)
        tgt[rng.choice(len(tgt), len(idx), replace=False)] = ts[idx]
        return src, np.ascontiguousarray(tgt), np.ascontiguousarray(ts)
    if kind == "outliers":                           # 0.1 % far outliers: dead columns at scale
        tgt = tgt.copy()
        k = max(1, len(tgt) // 1000)
        tgt[rng.choice(len(tgt), k, replace=False)] += rng.uniform(2.0, 5.0, (k, tgt.shape[1]))
        return src, tgt, ts
    raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------------------------------
# case bodies (shared by the H100 tests and their emulation-size runs)
# ---------------------------------------------------------------------------------------------------------------------------
def body_square(n, sigmas, ws=(0.0, 0.1), kinds=(None,), kind="rigid", dim=3):
    for var in kinds:
        src, tgt, ts = pair(n, kind=kind, dim=dim)
        if var is not None:
            src, tgt, ts = variant(src, tgt, ts, var)
        for s2 in sigmas:
            for w in ws:
                run_case("%dx%d %s%s s2=%g w=%g" % (n, n, kind, "" if var is None else " " + var, s2, w), src, tgt, ts, s2, w, dim=dim)


def body_shards(n, ranks_list, s2, w):
    """Shards of the targets as single handles with n_global: the first and the last rank against the reference; every rank's
    pt1 and the sum over the ranks of p1 against the single handle's reference (columns are separable, so the single handle's
    bound bounds the sum of the shards' errors)."""
    src, tgt, ts = pair(n)
    origin = tgt.mean(0)
    _, ref_all = run_case("%dx%d single s2=%g w=%g" % (n, n, s2, w), src, tgt, ts, s2, w, origin=origin)
    b_pt1, b_p1, _ = bounds(ref_all, ts)
    for ranks in ranks_list:
        cuts = [n * r // ranks for r in range(ranks + 1)]
        p1_sum = np.zeros(n)
        for r in range(ranks):
            lo, hi = cuts[r], cuts[r + 1]
            if r in (0, ranks - 1):
                (pt1, p1, px, n_p), ref = run_case("%d x shard %d/%d s2=%g w=%g" % (n, r, ranks, s2, w), src, tgt[lo:hi], ts, s2, w,
                                                   n_global=n, origin=origin)
            else:
                hs = handle_pair(3, src, tgt[lo:hi], n, origin)
                pt1, p1, px, n_p = hs[0].estep(ts, s2, w)
                for h in hs:
                    h.close()
            assert worst(pt1, ref_all.es.pt1[lo:hi], b_pt1[lo:hi], ~ref_all.extras.band[lo:hi]) <= 1.0
            p1_sum += p1
        assert worst(p1_sum, ref_all.es.p1, b_p1 + 2.0 ** -125 * ranks) <= 1.0, "%d shards: sum of p1" % ranks


def body_ragged(sizes, s2, w):
    for m, n in sizes:
        src, _, ts = pair(m)
        _, tgt, _ = pair(n)
        run_case("ragged %dx%d s2=%g w=%g" % (m, n, s2, w), src, tgt, ts, s2, w)


def body_bcpd(n, s2, w, seed=3):
    src, tgt, ts = pair(n)
    rng = np.random.default_rng(seed)
    alpha = rng.dirichlet(np.full(n, 2.0))
    sdiag = rng.uniform(0.0, 2.0 * s2, n)
    scale = 1.05
    origin = tgt.mean(0)
    hs = handle_pair(3, src, tgt, n, origin)
    outs = [h.bcpd_estep(ts, scale, alpha, sdiag, s2, w) for h in hs]
    for h in hs:
        h.close()
    ref = so.bcpd_expectation_step(ts, tgt, scale, alpha, sdiag, s2, w, frame_origin=origin, pair_err=_delta_wgt)
    la, _ = so.bcpd_exponents(alpha, sdiag, scale, s2, w, 3, True)
    assert 5.0 < la.max() < 60.0                       # a moderate but real span of per-source weights
    check_outputs("bcpd %dx%d s2=%g w=%g" % (n, n, s2, w), outs, ref, ts, bcpd=True)


def body_loop(n, s2, w):
    """The E-step inside cpd_em_step (captured graph on the device): step 1 at T_init, step 2 (a replay) at step 1's output."""
    src, tgt, _ = pair(n)
    origin = tgt.mean(0)
    rot, t, scale = orc.rot_z(29.5), TRUE_T.copy(), 1.0
    hs = handle_pair(3, src, tgt, n, origin)
    for step in (1, 2):
        for h in hs:       # step 2: the first step's transform at the same sigma2 (same graph key: the captured graph is replayed)
            h.set_state(_cabi.TF_RIGID, True, w, rot, t, scale, s2, 0.0)
        ts = orc.apply_rigid(src, rot, t, scale)
        res = [h.em_step() for h in hs]
        outs = [h.last_estep() for h in hs]
        anorm = float(np.sqrt((so.pack_coordinates(ts, s2, origin) ** 2).sum(1)).max())
        ref = so.expectation_step(ts, tgt, s2, w, frame_origin=origin, pair_err=_delta_loop(anorm))
        check_outputs("em_step %d %dx%d s2=%g w=%g" % (step, n, n, s2, w), outs, ref, ts)
        assert res[0][3] == res[1][3]
        rot, t, scale = res[0][0], res[0][1], res[0][2]
    for h in hs:
        h.close()


def sharpness(n, s2, w):
    """The same GPU outputs against references that are wrong by a little: the bound must see it."""
    src, tgt, ts = pair(n)
    origin = tgt.mean(0)
    h = handle_pair(3, src, tgt, n, origin)
    pt1, p1, px, n_p = h[0].estep(ts, s2, w)
    for x in h:
        x.close()
    good = so.expectation_step(ts, tgt, s2, w, frame_origin=origin, pair_err=_delta_plain)
    _, b_p1, _ = bounds(good, ts)
    assert worst(p1, good.es.p1, b_p1) <= 1.0
    # 1. the unrounded reference: the FP32 packing of the coordinates is 1 ulp of a_m, b_n away
    plain = so.expectation_step(ts, tgt, s2, w)
    q_plain = worst(p1, plain.es.p1, b_p1)
    # 2. K off by 2^-12 relative in every other source row
    pert = so.expectation_step(ts, tgt, s2, w, frame_origin=origin, pair_err=_delta_plain, k_scale=lambda rows: 1.0 + 2.0 ** -12 * (rows & 1))
    q_pert = worst(p1, pert.es.p1, b_p1)
    print("sharpness %dx%d s2=%g w=%g: worst err/bound against the unrounded reference %.1f, against K * (1 + 2^-12 [m odd]) %.1f"
          % (n, n, s2, w, q_plain, q_pert))
    assert q_plain > 1.0 and q_pert > 1.0


# ---------------------------------------------------------------------------------------------------------------------------
# the H100 tests
# ---------------------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


@gpu
@pytest.mark.timeout(900)
def test_bench_shape_100k():
    """bench.py's 1-GPU shape (98 pass-1 tiles, one wave) and the data variants."""
    body_square(100000, (1e-5, 1e-6))
    body_square(100000, (1e-5,), ws=(0.1,), kinds=("shift", "grid", "outliers"))


@gpu
@pytest.mark.timeout(900)
def test_bench_shards_2_4_8():
    """bench.py's 2/4/8-GPU shards (49 / 25 / 13 tiles, last-tile cost 0.875 / 0.5 / 0.25) as single handles with n_global."""
    body_shards(100000, (2, 4, 8), 1e-5, 0.1)


@gpu
@pytest.mark.timeout(900)
def test_config3_affine_250k_and_config4_shard():
    body_square(250000, (1e-6,), ws=(0.1,), kind="affine")
    src, tgt, ts = pair(1000000)
    lo, hi = 3 * 125000, 4 * 125000
    run_case("1M x shard 3/8 s2=1e-6 w=0.1", src, tgt[lo:hi], ts, 1e-6, 0.1, n_global=1000000, origin=tgt.mean(0))


@gpu
@pytest.mark.timeout(900)
def test_1m_square_several_waves():
    """977 pass-1 tiles: the several-waves branch of build_work on hardware, and pass 2 over 1M sources."""
    body_square(1000000, (1e-6,), ws=(0.1,))


@gpu
@pytest.mark.timeout(900)
def test_ragged_2d_bcpd_and_loop():
    a, b, c = 98 * 1024 - 1, 98 * 1024 + 1, 2 ** 17 + 1
    body_ragged(((a, b), (b, c), (c, a)), 1e-6, 0.1)
    body_square(200000, (1e-6,), ws=(0.0, 0.1), dim=2)
    body_bcpd(100000, 1e-5, 0.1)
    body_loop(100000, 1e-5, 0.1)


@gpu
@pytest.mark.timeout(600)
def test_bound_is_sharp():
    sharpness(100000, 1e-6, 0.1)


# ---------------------------------------------------------------------------------------------------------------------------
# the same bodies at sizes the CPU emulation runs (test logic, index and plan logic; not MUFU, not real races)
# ---------------------------------------------------------------------------------------------------------------------------
def test_bodies_at_emulation_size(emulated, monkeypatch):
    monkeypatch.setenv("CPD_EMU_SMS", "1")          # 2 resident CTAs per pass: every plan below has several waves
    body_square(2500, (1e-4, 1e-5), ws=(0.0, 0.1))
    body_square(2000, (1e-4,), ws=(0.1,), kinds=("shift", "grid", "outliers"))
    body_shards(2600, (2, 4), 1e-4, 0.1)
    body_ragged(((1023, 1025), (1025, 2049)), 1e-4, 0.1)
    body_square(2500, (1e-5,), ws=(0.1,), dim=2)
    body_bcpd(2000, 1e-4, 0.1)
    body_loop(2000, 1e-4, 0.1)


def test_sharpness_at_emulation_size(emulated, monkeypatch):
    monkeypatch.setenv("CPD_EMU_SMS", "2")
    sharpness(2500, 1e-5, 0.1)


def teardown_module(module):
    if ROWS:
        print("\ncase | instantiation | pairs | worst err / bound: pt1 | p1 | px")
        for r in ROWS:
            print("%s | %s | %.2e | %.3f | %.3f | %.3f" % r)
