"""Exact float64 E-steps by neighbour search  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The dense oracles (``cpd_oracle.expectation_step``, ``estep_oracle.c``) walk all M x N pairs, which is out of reach at the
sizes the benchmark measures (1e10 pairs at 100k^2, 1e12 at 1M^2).  At small sigma almost every pair is exactly zero in the
reference's own float64 arithmetic, so the same quantities can be formed from the pairs that are not:

* ``exp(-x)`` is exactly 0 in float64 for x > 745.2 (natural units; 1075 in log2 units), so such a pair contributes
  nothing to ``cpd.py:76-87`` (the column is dead when every pair is such a pair).
* Of the other pairs, per target n, only those with ``u_mn <= u_n,nearest + R`` are kept (log2 units, R = ``R_LOG2``).
  R is set by what the pair kernels can hold, not by float64 alone: the kernels evaluate 2^(o_n - u_mn) with an integer
  offset o_n that may sit up to 100 above the column's smallest u (pass 1's slow path fires at 2^100) and flush results
  below 2^-126 (``ex2.approx.ftz``), so a term 2^-226 of the column's largest may still be non-zero on the device.  Such a
  term is below 2^-125 of the column's largest P, which the tests' bound carries as an absolute term per kept pair.  With
  R = 160 every omitted term is below 2^-160 of the column's largest P: at most 2^21 of them per source row (the largest
  cloud tested) add up to < 2^-139, far under that absolute term.  160 log2 units are 110.9 natural units.

Two modes:

* ``frame_origin=None``: the reference's arithmetic on the caller's float64 coordinates (``K = exp(-d^2 / 2 sigma^2)``).
* ``frame_origin`` given: the reference's arithmetic on the kernel's own FP32 inputs.  ``pack_kernel`` forms, in FP64 with
  one final rounding, ``a_m = fl32(sk (ts_m - c_x))``, ``b_n = fl32(sk (x_n - c_x))``, ``sk = sqrt(LOG2E / (2 sigma^2))``,
  and ``c_x`` is exactly the origin handed to ``cpd_set_target``; numpy reproduces those floats bit for bit.  Then
  ``u_mn = |a_m - b_n|^2`` in float64, ``K = 2^-u``, and ``px_m = p1_m ts_m + sum_n P_mn (b_n - a_m) / sk`` -- the form
  ``finalize2_kernel`` / ``uncentre_px_kernel`` evaluate.

Besides the E-step the functions return the per-element sums an error bound needs (``Extras``): for every kept pair a
caller-chosen error weight ``delta_mn`` (``pair_err(u, la, col_umin)``, log2 units; default ``u``) is averaged per column with
the weights K (``col_dbar``) and summed per row with the weights P (``row_pd``, ``row_pdbar`` = sum_n P_mn col_dbar_n).
``row_sub`` is the absolute error pass 2 may make on the pairs of columns whose factor rn may leave float32's normal range.
"""
from collections import namedtuple

import numpy as np
from scipy.spatial import cKDTree

from oracle import cpd_oracle as orc

LOG2E = 1.4426950408889634074
R_LOG2 = 160.0                       # kept: u <= u_nearest + R_LOG2 (log2 units); see the module docstring
U_DEAD_LOG2 = 746.0 * LOG2E          # exp(-x) == 0 in float64 beyond x = 745.13 natural units
BAND_NAT = (690.0, 760.0)            # nearest exponent (natural units) in float64's denormal range: the reference is noisy there

Extras = namedtuple("Extras", ["pairs", "row_cnt", "col_cnt", "col_umin", "col_dbar", "row_pd", "row_pdbar", "row_sub", "dmax", "band"])
SparseEstep = namedtuple("SparseEstep", ["es", "extras"])


def pack_coordinates(points, sigma2, frame_origin):
    """``pack_kernel``'s FP32 coordinates in the sigma-scaled frame: fl32(sk (p - c_x)), returned as float64."""
    sk = np.sqrt(LOG2E / (2.0 * sigma2))
    return (sk * (np.asarray(points, dtype=np.float64) - np.asarray(frame_origin, dtype=np.float64))).astype(np.float32).astype(np.float64)


def _frames(t_source, target, sigma2, frame_origin):
    """(source points, target points, f) with u (log2 units) = f |p_m - q_n|^2, and sk (rounded mode) or None."""
    if frame_origin is None:
        return np.asarray(t_source, dtype=np.float64), np.asarray(target, dtype=np.float64), LOG2E / (2.0 * sigma2), None
    a = pack_coordinates(t_source, sigma2, frame_origin)
    b = pack_coordinates(target, sigma2, frame_origin)
    return a, b, 1.0, np.sqrt(LOG2E / (2.0 * sigma2))


def _sweep(p, q, f, la, chunk, per_chunk):
    """Neighbour search: per target chunk, the kept pairs (rows, cols, u in log2 units) handed to
    per_chunk(j0, rows, cols, u, col_umin).
    la (None or per-source exponent >= 0, log2 units) is added to u for the cut.  Returns (col_umin, pairs)."""
    n = q.shape[0]
    tree = cKDTree(p)
    dnn, inn = tree.query(q)
    umin = f * dnn ** 2
    best = umin if la is None else umin + la[inn]          # >= the column's smallest u + la
    pairs = 0
    for j0 in range(0, n, chunk):
        qb = q[j0:j0 + chunk]
        cut = best[j0:j0 + chunk] + R_LOG2
        r = np.sqrt(np.minimum(U_DEAD_LOG2, cut) / f) * (1.0 + 1e-9)
        lists = tree.query_ball_point(qb, r)
        lens = np.fromiter((len(x) for x in lists), np.int64, len(lists))
        rows = np.concatenate([np.asarray(x, np.int64) for x in lists]) if lens.sum() else np.zeros(0, np.int64)
        cols = np.repeat(np.arange(len(qb)), lens)
        u = f * ((p[rows] - qb[cols]) ** 2).sum(1)
        tot = u if la is None else u + la[rows]
        keep = (u <= U_DEAD_LOG2) & (tot <= cut[cols])
        rows, cols, u = rows[keep], cols[keep], u[keep]
        pairs += rows.size
        per_chunk(j0, rows, cols, u, umin[j0 + cols])
    return umin, pairs


class _Acc(object):
    """Per-row / per-column accumulators shared by both E-steps."""

    def __init__(self, m, n, dim):
        self.pt1, self.p1, self.px = np.zeros(n), np.zeros(m), np.zeros((m, dim))
        self.row_cnt, self.col_cnt = np.zeros(m, np.int64), np.zeros(n, np.int64)
        self.col_dbar, self.row_pd, self.row_pdbar, self.row_sub = np.zeros(n), np.zeros(m), np.zeros(m), np.zeros(m)
        self.umax = 0.0

    def add(self, j0, nb, rows, cols, k, den, delta, u, qv, pv, sk, ts, col_umin, la_free=True):
        m = self.p1.shape[0]
        # Pass 2 multiplies 2^(o - u) by rn = 2^-o / den in float32, and the offset o may sit up to 101 above the column's smallest u:
        # rn >= 2^-101 Pmax (Pmax = 2^-u_min / den bounds the column's largest P).  Where Pmax < 2^-25, rn may lie below float32's
        # normal range, keeping only an absolute 2^-149 (or flushing to 0): P_mn is then off by up to min(P_mn, 2^(o - u) 2^-150)
        # <= 2^-(u - u_min) min(Pmax, 2^-49) (without the per-source exponents; with them, the factor is 1).
        pmax = np.exp2(-col_umin) / den[cols]
        weak = pmax < 2.0 ** -25
        fac = np.exp2(-(u[weak] - col_umin[weak])) if la_free else 1.0
        self.row_sub += np.bincount(rows[weak], fac * np.minimum(pmax[weak], 2.0 ** -49), m)
        ksum = np.bincount(cols, k, nb)
        with np.errstate(invalid="ignore", divide="ignore"):
            dbar = np.where(ksum > 0, np.bincount(cols, k * delta, nb) / np.where(ksum > 0, ksum, 1.0), 0.0)
        pr = k / den[cols]
        self.pt1[j0:j0 + nb] = np.bincount(cols, pr, nb)
        self.p1 += np.bincount(rows, pr, m)
        if sk is None:
            for a in range(self.px.shape[1]):
                self.px[:, a] += np.bincount(rows, pr * qv[cols, a], m)
        else:                                   # p1 ts + sum P (b - a) / sk: the first part is added at the end
            for a in range(self.px.shape[1]):
                self.px[:, a] += np.bincount(rows, pr * (qv[cols, a] - pv[rows, a]), m) / sk
        self.row_cnt += np.bincount(rows, None, m).astype(np.int64)
        self.col_cnt[j0:j0 + nb] = np.bincount(cols, None, nb).astype(np.int64)
        self.col_dbar[j0:j0 + nb] = dbar
        self.row_pd += np.bincount(rows, pr * delta, m)
        self.row_pdbar += np.bincount(rows, pr * dbar[cols], m)
        if rows.size:
            self.umax = max(self.umax, float(u.max()))

    def finish(self, ts, sk, sigma2, umin, pairs):
        if sk is not None:
            self.px += self.p1[:, None] * ts
        dmax = np.sqrt(self.umax / (LOG2E / (2.0 * sigma2)))      # largest |a_m - b_n| / sk of a kept pair: a distance
        band = (umin / LOG2E > BAND_NAT[0]) & (umin / LOG2E < BAND_NAT[1])
        return Extras(pairs, self.row_cnt, self.col_cnt, umin, self.col_dbar, self.row_pd, self.row_pdbar, self.row_sub, dmax, band)


def _default_err(u, la, col_umin):
    return u


def expectation_step(t_source, target, sigma2, w, n_global=None, frame_origin=None, pair_err=None, k_scale=None, chunk=20000):
    """``cpd_oracle.expectation_step`` (cpd.py:71-88) over the kept pairs.  Returns SparseEstep(Estep, Extras).
    ``k_scale(rows)``: a factor applied to every K of those source rows (a deliberately wrong reference, for sharpness tests)."""
    ts = np.asarray(t_source, dtype=np.float64)
    tgt = np.asarray(target, dtype=np.float64)
    m, dim = ts.shape
    n = tgt.shape[0]
    c = orc.outlier_constant(sigma2, w, m, n if n_global is None else n_global, dim)
    p, q, f, sk = _frames(ts, tgt, sigma2, frame_origin)
    pair_err = pair_err or _default_err
    acc = _Acc(m, n, dim)

    def per_chunk(j0, rows, cols, u, col_umin):
        nb = min(chunk, n - j0)
        if sk is None:       # the reference's own expression: exp(-d^2 / (2 sigma^2))
            k = np.exp(-((p[rows] - q[j0 + cols]) ** 2).sum(1) / (2.0 * sigma2))
        else:
            k = np.exp2(-u)
        if k_scale is not None:
            k = k * k_scale(rows)
        den = np.bincount(cols, k, nb)
        den[den == 0] = orc.EPS32                              # cpd.py:81
        den += c                                               # cpd.py:82
        acc.add(j0, nb, rows, cols, k, den, pair_err(u, None, col_umin), u, q[j0:j0 + nb], p, sk, ts, col_umin)

    umin, pairs = _sweep(p, q, f, None, chunk, per_chunk)
    return SparseEstep(orc.Estep(acc.pt1, acc.p1, acc.px, float(acc.p1.sum())), acc.finish(ts, sk, sigma2, umin, pairs))


def bcpd_exponents(alpha, sigma_diag, scale, sigma2, w, dim, rounded):
    """Per-source exponents of the weighted E-step (log2 units) as ``bcpd_la_kernel`` / ``bcpd_la_apply_kernel`` form them:
    la_m = -log2(alpha_m) - log2(1 - w) + scale^2 / (2 sigma2) D log2(e) Sigma_mm in FP64, then la_m - la_min (float32 when
    rounded, capped at 1e30).  Returns (la' (float64 array), la_min)."""
    alpha = np.asarray(alpha, dtype=np.float64)
    sdiag = np.asarray(sigma_diag, dtype=np.float64)
    kf = scale * scale / (2.0 * sigma2) * float(dim) * LOG2E
    with np.errstate(divide="ignore"):
        la = np.where(alpha > 0.0, -np.log2(np.where(alpha > 0.0, alpha, 1.0)), np.inf) + (-np.log2(1.0 - w)) + kf * sdiag
    la_min = float(la.min())
    rel = np.minimum(la - la_min, 1.0e30)
    if rounded:
        rel = rel.astype(np.float32).astype(np.float64)
    return rel, la_min


def bcpd_expectation_step(t_source, target, scale, alpha, sigma_diag, sigma2, w, n_global=None, frame_origin=None, pair_err=None,
                          chunk=20000):
    """``cpd_oracle.bcpd_expectation_step`` (bcpd.py:53-72) over the kept pairs: the cut is u + la'_m <= best + R with best
    bounded by the nearest source's u + la'.  Returns SparseEstep(Estep(nu_d, nu, px, n_p), Extras)."""
    ts = np.asarray(t_source, dtype=np.float64)
    tgt = np.asarray(target, dtype=np.float64)
    m, dim = ts.shape
    n = tgt.shape[0]
    ng = n if n_global is None else n_global
    p, q, f, sk = _frames(ts, tgt, sigma2, frame_origin)
    la, la_min = bcpd_exponents(alpha, sigma_diag, scale, sigma2, w, dim, sk is not None)
    pair_err = pair_err or _default_err
    acc = _Acc(m, n, dim)
    alpha = np.asarray(alpha, dtype=np.float64)
    sdiag = np.asarray(sigma_diag, dtype=np.float64)
    lognorm = (2.0 * np.pi * sigma2) ** (dim * 0.5)
    wfac = np.exp(-(scale ** 2) / (2.0 * sigma2) * sdiag * dim) * (1.0 - w) * alpha          # bcpd.py:57-63
    # kernel units: phi = 2^-(u + la') 2^-la_min / (2 pi sigma2)^(D/2);  den / that factor = sum 2^-(u + la') + c'
    c_rounded = (w / ng) * 2.0 ** la_min * lognorm

    def per_chunk(j0, rows, cols, u, col_umin):
        nb = min(chunk, n - j0)
        if sk is None:
            d2 = ((p[rows] - q[j0 + cols]) ** 2).sum(1)
            k = np.exp(-d2 / (2.0 * sigma2)) / lognorm * wfac[rows]
            den = w / ng + np.bincount(cols, k, nb)
        else:
            k = np.exp2(-(u + la[rows]))
            den = np.bincount(cols, k, nb) + c_rounded
        den[den == 0] = orc.EPS32
        acc.add(j0, nb, rows, cols, k, den, pair_err(u, la[rows], col_umin), u, q[j0:j0 + nb], p, sk, ts, col_umin, la_free=False)

    umin, pairs = _sweep(p, q, f, la, chunk, per_chunk)
    return SparseEstep(orc.Estep(acc.pt1, acc.p1, acc.px, float(acc.p1.sum())), acc.finish(ts, sk, sigma2, umin, pairs))
