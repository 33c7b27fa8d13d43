"""The G X products of the low-rank range finder, element by element (cpd_lowrank_gram_product).

G_ij = exp(-|y_i - y_j|^2 / 2 beta) is never stored: the exact integer-digit tensor-core kernel (csrc/gram_i8.cuh) and the
CUDA-core kernel (csrc/lowrank.cuh) generate it tile by tile.  The tests here look at single elements of G X:

  a. coincident clusters far apart, X on a 2^-22 grid: G is exactly 0 / 1, every digit and every FP32 partial sum is exact, so
     both kernels must return the cluster sums bit for bit -- at the row-tile, column-pass and j-chunk edges;
  b. identities that hold bit for bit on any cloud: a column of G X does not depend on the other columns, and the row shares of a
     multi-rank handle add up to the whole product;
  c. smooth clouds against G X in float64, within a tolerance derived from the arithmetic (_tolerance), which a numpy model of
     the digit product shows to reject a missing stage, a dropped MMA and swapped columns;
  d. a full j-chunk where every digit is near its extreme: the int32 accumulators of the tensor-core kernel at their bound.

The CPU emulation has no tensor-core kernel: the emulated tests run the CUDA-core kernel at small sizes.
"""
import math

import numpy as np
import pytest

from probreg_b200 import _cabi
from test_zz_lowrank import _deformed_pair

TC, CC = _cabi.Handle.GRAM_TENSOR_CORES, _cabi.Handle.GRAM_CUDA_CORES
NAMES = {TC: "tensor cores", CC: "CUDA cores"}
LOG2E = 1.4426950408889634
U = 2.0 ** -24                     # unit round-off of float32


def _handle(src, beta):
    """A handle after a low-rank set-up with `beta` on `src` (rank 1, no power iteration: only beta and the points matter)."""
    h = _cabi.Handle(src.shape[1])
    h.set_source(src)
    h.set_target(src[:64])
    h.nonrigid_lowrank_begin(beta, 2.0, 0.1, 0.0, 1, 0, 1)
    return h


# ---- a. coincident clusters: exact -----------------------------------------------------------------------------------------------
CLUSTER_BETA = 1.0
CLUSTER_SPACING = 20.0             # scaled u = 20^2 log2(e) / (2 beta) = 288 > 160 between clusters: ex2 gives exactly 0


def _clusters(m, dim, seed):
    """m points in coincident clusters of 1 .. 300 points on a grid of CLUSTER_SPACING; (points, cluster label per point)."""
    rng = np.random.default_rng(seed)
    sizes, total = [], 0
    for s in [1, 1, 2, 300, 3] + list(rng.integers(1, 301, size=m)):
        s = min(int(s), m - total)
        sizes.append(s)
        total += s
        if total == m:
            break
    ncl = len(sizes)
    side = int(math.ceil(ncl ** (1.0 / dim))) + 1
    grid = np.stack(np.meshgrid(*[np.arange(side)] * dim, indexing="ij"), -1).reshape(-1, dim)[:ncl] * CLUSTER_SPACING
    lab = np.repeat(np.arange(ncl), sizes)
    rng.shuffle(lab)
    return grid[lab] + 0.25, lab


def _grid_columns(m, cols, rng):
    """Columns k 2^-22, |k| <= 2^19, with one entry of exactly 2^19: the column maximum is 2^-3, the i8 digits are exact, and
    so are the float32 values and 32-term float32 sums of the CUDA-core kernel.  From 4 columns on, the last three are special:
    all zero, a single nonzero entry, and a maximum of negative sign."""
    k = rng.integers(-2 ** 19, 2 ** 19 + 1, size=(m, cols))
    k[rng.integers(0, m, size=cols), np.arange(cols)] = 2 ** 19
    x = k * 2.0 ** -22
    if cols >= 4:
        x[:, -3] = 0.0
        x[:, -2] = 0.0
        x[rng.integers(0, m), -2] = float(np.float32(-0.3))
        kn = rng.integers(-2 ** 19 + 1, 2 ** 19, size=m)
        kn[rng.integers(0, m)] = -2 ** 19
        x[:, -1] = kn * 2.0 ** -22
    return x


def _cluster_sums(x, lab):
    order = np.argsort(lab, kind="stable")
    starts = np.flatnonzero(np.r_[True, np.diff(lab[order]) != 0])
    sums = np.add.reduceat(x[order], starts, axis=0)          # exact: multiples of 2^-22 below 2^6
    return sums[lab]


def _check_clusters(ms, cols_list, dims, kernels):
    for dim in dims:
        for m in ms:
            pts, lab = _clusters(m, dim, seed=m + dim)
            h = _handle(pts, CLUSTER_BETA)
            rng = np.random.default_rng(m)
            for cols in cols_list:
                x = _grid_columns(m, cols, rng)
                want = _cluster_sums(x, lab)
                for kern in kernels:
                    got = h.lowrank_gram_product(x, kern)
                    bad = np.argwhere(got != want)
                    assert bad.size == 0, (NAMES[kern], dim, m, cols, len(bad), bad[:5].tolist())


def test_cluster_sums_are_exact_emulated(emulated):
    _check_clusters([1, 31, 127, 128, 129, 511, 513], [1, 16, 17, 63, 64, 65], (3,), (CC,))
    _check_clusters([129, 600], [17, 130], (2,), (CC,))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_cluster_sums_are_exact_gpu():
    """Both kernels, M from one row through row tiles (128), the first two-chunk size with a 512-point last chunk (16385), more
    than one unit per CTA (133+ tiles), three chunks with a ragged last one (40000) to configuration 5 (50000); 1 .. 200 columns
    (one to four column passes of 64)."""
    _check_clusters([1, 31, 127, 128, 129, 511, 513, 16384, 16385, 17000, 40000, 50000], [1, 16, 17, 63, 64, 65, 130, 200], (3,),
                    (TC, CC))
    _check_clusters([129, 16385, 40000], [17, 130], (2,), (TC, CC))


# ---- b. identities that hold bit for bit -----------------------------------------------------------------------------------------
def _smooth_columns(m, cols, seed):
    """Standard normal columns, column 0 constant (every row of G X is then nonzero)."""
    x = np.random.default_rng(seed).standard_normal((m, cols))
    x[:, 0] = 1.0
    return x


def _check_identities(m, kernels):
    src, _ = _deformed_pair(m)
    h = _handle(src, 2.0)
    x = _smooth_columns(m, 200, seed=5)
    for kern in kernels:
        full = h.lowrank_gram_product(x, kern)
        # a column does not depend on the columns around it, nor on the pass it falls in
        for sel in (np.arange(60, 70), np.array([5, 63, 64, 127, 128, 199]), np.arange(190, 200), np.array([129])):
            assert np.array_equal(h.lowrank_gram_product(x[:, sel], kern), full[:, sel]), (NAMES[kern], sel)
        # the row shares of a multi-rank handle: contiguous shares of the internal order, m r / world .. m (r + 1) / world
        for world in (2, 3, 8):
            parts = [h.lowrank_gram_product(x, kern, world=world, rank=r) for r in range(world)]
            filled = np.array([np.any(p != 0.0, axis=1) for p in parts])
            assert np.all(filled.sum(0) == 1), (NAMES[kern], world)
            assert [int(f.sum()) for f in filled] == [m * (r + 1) // world - m * r // world for r in range(world)]
            assert np.array_equal(np.sum(parts, axis=0), full), (NAMES[kern], world)
            for p, f in zip(parts, filled):
                assert np.array_equal(p[f], full[f]) and not np.any(p[~f])


def test_column_and_shard_identities_emulated(emulated):
    _check_identities(700, (CC,))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_column_and_shard_identities_gpu():
    _check_identities(17000, (TC, CC))


# ---- c. smooth clouds against float64 --------------------------------------------------------------------------------------------
def _tolerance(src, beta, x, rows, kernels):
    """Per-element bounds on |kernel(G X) - G64 X| for the rows `rows`; returns (G64 X, {kernel: bound}).

    Both kernels evaluate the same float32 G:  a = fl(sb fl(y)), sb = fl(sqrt(log2 e / 2 beta)),  u = |a_i - a_j|^2 by an FMA chain
    on float32 differences,  e = ex2.approx(-u).  Against G64 = 2^-u64 (u64 exact):
      - coordinates: |a - sb y| <= 2^-23 A (two roundings; A = sb max |y|), so each difference moves by <= 2^-22 A and
        |du| <= 2^-21 A sqrt(D u) + D 2^-44 A^2;
      - the float32 u: 3 subtractions, 3 products / FMAs, and sb squared: |du| <= 8 2^-24 u;
      - ex2.approx: 2 ulp, 2^-22 relative; results below 2^-126 flush to 0;
    so t1 = 1.01 (G64 (2^-22 + ln 2 |du|) + 2^-126)  (1.01: second-order terms).
    Tensor cores (gram_i8.cuh): G X = colmax 2^-45 sum_j g_ij x_cj with g = round(2^23 e), x = round(2^22 X / colmax); then
      (1) sum_j t1_ij |X^_cj|                                       the float32 G, |X^| <= |X| + 2^-23 colmax
      (2) 2^-24 sum_j |X^_cj|                                      rounding g
      (3) 2^-23 colmax_c sum_j (G64_ij + t1_ij + 2^-24)             rounding x, against g 2^-23 <= e + 2^-24
      (4) colmax_c 2^-45 sum_j (2^15 (a1 + a2) + 2^7 a2)           the dropped levels 3 and 4: a1 b2 + a2 b1 at 2^8, a2 b2 at 1,
                                                                   |b| <= 128, a1 <= min(255, g / 2^8), a2 <= min(255, g)
      plus 2^-50 sum_j G64 |X| for the FP64 sum of the chunk partials.
    CUDA cores (lowrank.cuh): (1), then X rounded to float32 (2^-24 relative), 32-term float32 FMA sums (31 roundings: 32 2^-24 of
    the sum of |terms|) and the FP64 sum of the m / 32 group sums."""
    m, dim = src.shape
    sb = math.sqrt(LOG2E / (2.0 * beta))
    a_max = sb * np.abs(src).max()
    ax = np.abs(x)
    colmax = ax.max(0)
    want = np.empty((len(rows), x.shape[1]))
    tol = {k: np.empty_like(want) for k in kernels}
    for b0 in range(0, len(rows), 256):
        r = rows[b0:b0 + 256]
        d2 = np.zeros((len(r), m))
        for k in range(dim):
            d2 += (src[r, k][:, None] - src[None, :, k]) ** 2
        u = d2 * (LOG2E / (2.0 * beta))
        g64 = np.exp2(-u)
        du = 8.0 * U * u + 2.0 ** -21 * a_max * np.sqrt(dim * u) + dim * 2.0 ** -44 * a_max ** 2
        t1 = 1.01 * (g64 * (2.0 ** -22 + math.log(2.0) * du) + 2.0 ** -126)
        want[b0:b0 + len(r)] = g64.dot(x)
        gx = g64.dot(ax)
        t1x = t1.dot(ax)
        if TC in kernels:
            xq = ax + 2.0 ** -23 * colmax                                    # |X^|
            gu = np.floor(2.0 ** 23 * (g64 + t1) + 0.5)                      # g <= gu
            a1, a2 = np.minimum(255.0, np.floor(gu / 256.0)), np.minimum(255.0, gu)
            lv34 = (2.0 ** 15 * (a1 + a2) + 2.0 ** 7 * a2).sum(1)
            tol[TC][b0:b0 + len(r)] = (t1x + 2.0 ** -23 * colmax * t1.sum(1)[:, None]                                  # (1)
                 + U * xq.sum(0)[None, :]                                                        # (2)
                 + 2.0 ** -23 * colmax[None, :] * (g64 + t1 + U).sum(1)[:, None]                 # (3)
                 + 2.0 ** -45 * colmax[None, :] * lv34[:, None]                                  # (4)
                 + 2.0 ** -50 * gx)
        if CC in kernels:
            ex = (gx + t1x) * (1.0 + U)                                      # sum_j e_ij |fl32(X_cj)|
            tol[CC][b0:b0 + len(r)] = t1x * (1.0 + U) + U * (gx + t1x) + (32.0 * U + 2.0 ** -53 * (m / 32.0 + 16.0)) * ex * (1.0 + 64.0 * U)
    return want, tol


def _check_fp64(m, betas, kernels, cols=70):
    """Every row of G X against float64 G64 X; the worst error / tolerance of each kernel is printed."""
    src, _ = _deformed_pair(m)
    x = _smooth_columns(m, cols, seed=11)
    rows = np.arange(m)
    worst = {}
    for beta in betas:
        h = _handle(src, beta)
        got = {k: h.lowrank_gram_product(x, k) for k in kernels}
        want, tol = _tolerance(src, beta, x, rows, kernels)
        for k in kernels:
            ratio = np.abs(got[k] - want) / tol[k]
            i, c = np.unravel_index(np.argmax(ratio), ratio.shape)
            worst[(k, beta)] = ratio[i, c]
            print("G X vs float64, %s, M = %d, beta = %g: worst |error| / tolerance = %.3g (row %d, column %d)"
                  % (NAMES[k], m, beta, ratio[i, c], i, c))
            assert ratio[i, c] <= 1.0, (NAMES[k], beta, i, c, got[k][i, c], want[i, c], tol[k][i, c])
        if len(kernels) == 2:          # the two kernels with each other, over all rows: within the sum of their bounds
            assert np.all(np.abs(got[TC] - got[CC]) <= tol[TC] + tol[CC]), beta
    return worst


def test_against_float64_emulated(emulated):
    _check_fp64(600, (0.05, 2.0, 50.0), (CC,))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_against_float64_gpu():
    """17000 points: two j-chunks (the second one ragged), 133 row tiles on 132 SMs; 70 columns: a full and a partial pass."""
    _check_fp64(17000, (0.05, 2.0, 50.0), (TC, CC))


def _digit_model(src, beta, x, drop_stage=None, drop_a2b0=False):
    """numpy model of gi_gram_kernel: float32 G as the kernel forms it (without FMA contraction), the digit split of gi_split_kernel,
    the six digit MMAs of levels 0-2 as exact integer products, the FP64 join."""
    sb = np.float32(math.sqrt(LOG2E / (2.0 * beta)))
    a = sb * src.astype(np.float32)
    u = np.zeros((len(src), len(src)), dtype=np.float32)
    for k in range(src.shape[1]):
        d = a[:, k][:, None] - a[None, :, k]
        u = u + d * d
    g = np.rint(np.exp2(-u).astype(np.float64) * 2.0 ** 23).astype(np.int64)
    if drop_stage is not None:
        g[:, drop_stage:drop_stage + 32] = 0
    a0, a1, a2 = g >> 16, (g >> 8) & 255, g & 255
    colmax = np.abs(x).max(0)
    xi = np.rint(x * (2.0 ** 22 / colmax)).astype(np.int64)
    b2 = ((xi + 128) & 255) - 128
    r1 = (xi - b2) >> 8
    b1 = ((r1 + 128) & 255) - 128
    b0 = (r1 - b1) >> 8
    l0 = a0.dot(b0)
    l1 = a0.dot(b1) + a1.dot(b0)
    l2 = a0.dot(b2) + a1.dot(b1) + (0 if drop_a2b0 else a2.dot(b0))
    return (l0.astype(np.float64) * 65536.0 + l1 * 256.0 + l2) * (colmax * 2.0 ** -29)


def test_tolerance_rejects_a_missing_stage_a_dropped_mma_and_swapped_columns():
    """The bound of _tolerance holds for a faithful numpy model of the tensor-core product and fails for three faults of the kind a
    wrong descriptor, barrier phase or epilogue index would cause (shown on the model, not by breaking a kernel)."""
    m = 1500
    src, _ = _deformed_pair(m)
    x = _smooth_columns(m, 8, seed=3)
    rows = np.arange(m)
    for beta in (0.05, 2.0, 50.0):
        want, tol = _tolerance(src, beta, x, rows, (TC,))
        tol = tol[TC]
        assert (np.abs(_digit_model(src, beta, x) - want) / tol).max() <= 1.0, beta
        missing = _digit_model(src, beta, x, drop_stage=736)
        assert (np.abs(missing - want) / tol).max() > 10.0, beta
        dropped = _digit_model(src, beta, x, drop_a2b0=True)
        assert (np.abs(dropped - want) / tol).max() > 10.0, beta
        swapped = _digit_model(src, beta, x)[:, [0, 2, 1, 3, 4, 5, 6, 7]]
        assert (np.abs(swapped - want) / tol).max() > 10.0, beta
    # the CUDA-core bound, on a float32 restatement of lr_gram_apply_kernel
    beta = 2.0
    want, tol = _tolerance(src, beta, x, rows, (CC,))
    tol = tol[CC]
    sb = np.float32(math.sqrt(LOG2E / (2.0 * beta)))
    a = sb * src.astype(np.float32)
    u = sum((a[:, k][:, None] - a[None, :, k]) ** 2 for k in range(3)).astype(np.float32)
    e = np.exp2(-u)
    xf = x.astype(np.float32)
    cc = sum(e[:, j0:j0 + 32].dot(xf[j0:j0 + 32]).astype(np.float64) for j0 in range(0, m, 32))
    assert (np.abs(cc - want) / tol).max() <= 1.0


# ---- d. the int32 accumulators at their bound -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_accumulator_headroom_at_a_full_chunk_gpu():
    """16384 points (one full j-chunk) in a ball where G >= 1 - 2^-10: the G digits are (127, >= 224, any).  X digits
    (-63, -128, -128) / (63, 127, 127) on every point but one, which holds the column maximum: each accumulator level adds
    one-signed products of up to 3 x 2^15 per point (the level-2 accumulator reaches 1.06e9 of the 2^31 that int32 holds)."""
    m, beta = 16384, 1.0
    rng = np.random.default_rng(21)
    v = rng.standard_normal((m, 3))
    v *= (0.02 * rng.random(m) ** (1.0 / 3.0) / np.linalg.norm(v, axis=1))[:, None]
    src = v + np.array([0.3, -0.2, 0.1])             # |y_i - y_j| <= 0.04: u <= 1.2e-3, G >= 0.9992 > 1 - 2^-10
    x = np.empty((m, 3))
    x[:, 0] = -4161664 * 2.0 ** -22                  # digits (-63, -128, -128) against a column maximum of 1
    x[:, 1] = 4161407 * 2.0 ** -22                   # digits (63, 127, 127)
    x[:, 2] = rng.choice([-1.0, 1.0], m) * 4161664 * 2.0 ** -22
    x[7, :] = [-1.0, 1.0, 1.0]
    h = _handle(src, beta)
    rows = np.arange(m)
    want, tol = _tolerance(src, beta, x, rows, (TC, CC))
    for k in (TC, CC):
        got = h.lowrank_gram_product(x, k)
        ratio = np.abs(got - want) / tol[k]
        print("full chunk at the digit extremes, %s: worst |error| / tolerance = %.3g" % (NAMES[k], ratio.max()))
        assert ratio.max() <= 1.0, NAMES[k]


# ---- the entry point itself ------------------------------------------------------------------------------------------------------
def _check_arguments(kernels):
    src, _ = _deformed_pair(300)
    h = _cabi.Handle(3)
    h.set_source(src)
    h.set_target(src)
    with pytest.raises(_cabi.CpdError, match="lowrank_begin"):
        h.lowrank_gram_product(np.ones((300, 2)), CC)                        # nothing begun
    h.nonrigid_begin(2.0, 2.0, 0.1, 0.0)
    with pytest.raises(_cabi.CpdError, match="lowrank_begin"):
        h.lowrank_gram_product(np.ones((300, 2)), CC)                        # the dense path has no packed points
    h.nonrigid_lowrank_begin(2.0, 2.0, 0.1, 0.0, 20, 1, 3)
    q, b = h.nonrigid_lowrank_factors()
    for bad in (dict(kernel=2), dict(kernel=-1), dict(kernel=CC, world=0), dict(kernel=CC, world=2, rank=2),
                dict(kernel=CC, world=3, rank=-1)):
        with pytest.raises(_cabi.CpdError):
            h.lowrank_gram_product(np.ones((300, 2)), **bad)
    for cols in (0, 1025):
        with pytest.raises(_cabi.CpdError):
            h.lowrank_gram_product(np.ones((300, cols)), CC)
    with pytest.raises(ValueError):
        h.lowrank_gram_product(np.ones((299, 2)), CC)
    for k in kernels:
        assert h.lowrank_gram_product(np.ones((300, 1024)), k).shape == (300, 1024)
    # the factors and the iteration are untouched
    q2, b2 = h.nonrigid_lowrank_factors()
    assert np.array_equal(q, q2) and np.array_equal(b, b2)
    h.set_target(src + 0.01)
    h.nonrigid_restart(2.0, 0.1, 0.0)
    s_after = [h.nonrigid_step() for _ in range(2)]
    ref = _cabi.Handle(3)
    ref.set_source(src)
    ref.set_target(src + 0.01)
    ref.nonrigid_lowrank_begin(2.0, 2.0, 0.1, 0.0, 20, 1, 3)
    assert s_after == [ref.nonrigid_step() for _ in range(2)]


def test_entry_point_arguments_emulated(emulated):
    _check_arguments((CC,))
    src, _ = _deformed_pair(100)
    with pytest.raises(_cabi.CpdError, match="no tensor-core"):
        _handle(src, 1.0).lowrank_gram_product(np.ones((100, 3)), TC)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_entry_point_arguments_gpu():
    _check_arguments((TC, CC))


# ---- two devices in one process --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lowrank_setup_on_two_devices_in_one_process():
    """The tensor-core kernel needs more than 48 KB of dynamic shared memory, an attribute CUDA keeps per device: set-ups on a
    second device of the same process must launch as well, and give what the first one gives."""
    if _cabi.lib().cpd_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    src, _ = _deformed_pair(3000)
    x = _smooth_columns(3000, 70, seed=1)
    out = []
    for dev in (0, 1, 0):
        h = _cabi.Handle(3, device=dev)
        h.set_source(src)
        h.set_target(src)
        h.nonrigid_lowrank_begin(2.0, 2.0, 0.1, 0.0, 100, 2, 7)
        out.append((h.nonrigid_lowrank_factors(), h.lowrank_gram_product(x, TC)))
    for (q, b), gx in out[1:]:
        assert np.array_equal(q, out[0][0][0]) and np.array_equal(b, out[0][0][1]) and np.array_equal(gx, out[0][1])
