"""FilterReg oracle (test infrastructure): what the reference probreg v0.3.7 computes, restated.

* ``ref_filter`` / ``ref_lattice_size`` call the reference's UNMODIFIED permutohedral lattice, compiled by
  ``oracle/permutohedral.mk`` into ``oracle/_ref/libpermutohedral_ref.so`` (``ref_available()`` tells whether it was built).
* ``lattice_filter`` is a numpy float32 restatement of the same lattice on x86-64 (permutohedral.cpp:139-325 SSE build, 482-616
  filter): every float operation separately rounded in the reference's order.  It is checked bit for bit against the compiled
  reference and is the specification the device build follows.  ``rounding="ties_down"`` and ``pad_lane=False`` restate two
  plausible mistakes (the scalar path's tie rule; forgetting the zero padding lanes of the 4-point blocks).
* ``expectation_step`` (filterreg.py:78-108), ``maximization_step`` (:159-196) and ``registration`` (:120-147) in FP64, with
  ``kabsch`` (cc/kabsch.cc:6-56), ``kabsch2d`` (:58-109) and ``compute_twist_for_pt2pl`` (cc/point_to_plane.cc:6-32).
* ``kabsch_f32`` / ``kabsch2d_f32`` / ``pt2pl_f32``: float32 restatements of the same C++ (what pybind11 hands the reference),
  used to record ``tests/golden/filterreg.npz``.
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libpermutohedral_ref.so")
_ref = None


def ref_available():
    return os.path.exists(REF_LIB)


def _lib():
    global _ref
    if _ref is None:
        _ref = ctypes.CDLL(REF_LIB)
        fp = ctypes.POINTER(ctypes.c_float)
        _ref.prl_filter.argtypes = [fp, ctypes.c_int, ctypes.c_int, fp, ctypes.c_int, ctypes.c_int, fp, ctypes.POINTER(ctypes.c_int)]
        _ref.prl_lattice_size.argtypes = [fp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return _ref


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def ref_filter(feature, values, with_blur=True):
    """(out (n x vs float32), lattice size) of the compiled reference: Permutohedral(feature, with_blur).filter(values)."""
    f = np.ascontiguousarray(feature, dtype=np.float32)
    v = np.ascontiguousarray(values, dtype=np.float32)
    if v.ndim == 1:
        v = v[:, None]
    out = np.empty_like(v)
    size = ctypes.c_int()
    assert _lib().prl_filter(_fp(f), f.shape[0], f.shape[1], _fp(v), v.shape[1], int(with_blur), _fp(out), ctypes.byref(size)) == 0
    return out, size.value


def ref_lattice_size(feature, with_blur=True):
    f = np.ascontiguousarray(feature, dtype=np.float32)
    return _lib().prl_lattice_size(_fp(f), f.shape[0], f.shape[1], int(with_blur))


# ---- numpy float32 restatement of the lattice ------------------------------------------------------------------------------
F = np.float32


def lattice_build(feature, with_blur=True, rounding="even", pad_lane=True):
    """Permutohedral::init (SSE path).  Returns (keys (P x (d+1) x d int16) of every elevated point incl. the padding lane,
    bary (n x (d+1) float32), n)."""
    f = np.asarray(feature, dtype=F)
    n, d = f.shape
    if pad_lane and n % 4:
        f = np.vstack([f, np.zeros((1, d), F)])          # the padding lanes of the last 4-point block, all the zero vector
    p = f.shape[0]
    inv_std = F(np.sqrt(2.0 / 3.0) * (d + 1)) if with_blur else F(np.sqrt(1.0 / 6.0) * (d + 1))
    sf = [F(1.0 / np.sqrt(float((i + 2) * (i + 1))) * float(inv_std)) for i in range(d)]
    invdp1, dp1 = F(1.0) / F(d + 1), F(d + 1)
    el = np.zeros((p, d + 1), F)
    sm = np.zeros(p, F)
    for j in range(d, 0, -1):
        cf = f[:, j - 1] * sf[j - 1]
        el[:, j] = sm - F(j) * cf
        sm = sm + cf
    el[:, 0] = sm
    v = invdp1 * el
    if rounding == "even":
        v = np.rint(v)
    else:                                                  # ties towards the lower multiple (the scalar path's rule, mis-applied)
        v = np.where(v - np.floor(v) == F(0.5), np.floor(v), np.rint(v)).astype(F)
    rem0 = v * dp1
    s = np.zeros(p, F)
    for i in range(d + 1):
        s = s + v[:, i]
    rank = np.zeros((p, d + 1), F)
    for i in range(d):
        di = el[:, i] - rem0[:, i]
        for j in range(i + 1, d + 1):
            c = (di < el[:, j] - rem0[:, j]).astype(F)
            rank[:, i] = rank[:, i] + c
            rank[:, j] = rank[:, j] + (F(1) - c)
    for i in range(d + 1):
        rank[:, i] = rank[:, i] + s
        a = np.where(rank[:, i] < 0, dp1, F(0)) - np.where(rank[:, i] >= dp1, dp1, F(0))
        rank[:, i] = rank[:, i] + a
        rem0[:, i] = rem0[:, i] + a
    b = np.zeros((p, d + 2), F)
    rows = np.arange(p)
    for i in range(d + 1):
        vv = (el[:, i] - rem0[:, i]) * invdp1
        q = d - rank[:, i].astype(np.int64)
        b[rows, q] = b[rows, q] + vv
        b[rows, q + 1] = b[rows, q + 1] - vv
    b[:, 0] = b[:, 0] + (F(1) + b[:, d + 1])
    ri = rank.astype(np.int64)
    keys = np.zeros((p, d + 1, d), np.int16)
    for r in range(d + 1):
        for i in range(d):
            canon = np.where(ri[:, i] <= d - r, r, r - (d + 1)).astype(F)
            keys[:, r, i] = (rem0[:, i] + canon).astype(np.int64).astype(np.int16)     # float -> int -> short, wrapping
    return keys, b[:n, :d + 1], n


def _pack(k):
    k = k.astype(np.int64) & 0xFFFF
    out = np.zeros(k.shape[:-1], np.int64)
    for i in range(k.shape[-1]):
        out |= k[..., i] << (16 * i)
    return out


def lattice_filter(feature, values, with_blur=True, rounding="even", pad_lane=True, sse=None):
    """(out (n x vs float32), lattice size) of the numpy restatement.  sse None: compute()'s dispatch (vs >= 3)."""
    keys, bary, n = lattice_build(feature, with_blur, rounding, pad_lane)
    d = keys.shape[2]
    v = np.asarray(values, dtype=F)
    if v.ndim == 1:
        v = v[:, None]
    vs = v.shape[1]
    sse = vs >= 3 if sse is None else sse
    packed = _pack(keys)
    ukey, inv = np.unique(packed.ravel(), return_inverse=True)
    nv = len(ukey)
    off = inv.reshape(packed.shape)[:n]                   # vertex of each real (point, remainder)
    vals = np.zeros((nv + 1, vs), F)                      # row 0: the zero row a missing neighbour reads
    # splat in (point, remainder) order; ufunc.at adds unbuffered, in index order
    np.add.at(vals, (off + 1).ravel(), (bary[:, :, None] * v[:, None, :]).reshape(-1, vs))
    if with_blur:
        uk = ((ukey[:, None] >> (16 * np.arange(d))) & 0xFFFF).astype(np.uint16).astype(np.int16).astype(np.int64)
        for j in range(d + 1):
            n1, n2 = uk - 1, uk + 1
            if j < d:
                n1[:, j], n2[:, j] = uk[:, j] + d, uk[:, j] - d
            nb = []
            for nk in (n1, n2):
                pk = _pack(nk.astype(np.int16))
                pos = np.clip(np.searchsorted(ukey, pk), 0, nv - 1)
                nb.append(np.where(ukey[pos] == pk, pos + 1, 0))
            old = vals[1:]
            sn = vals[nb[0]] + vals[nb[1]]
            new = np.zeros_like(vals)
            if sse:
                new[1:] = old + F(0.5) * sn
            else:
                new[1:] = (old.astype(np.float64) + 0.5 * sn.astype(np.float64)).astype(F)
            vals = new
    alpha = F(1) / (F(1) + F(2.0 ** -d))
    out = np.zeros((n, vs), F)
    for j in range(d + 1):
        w = bary[:, j][:, None]
        vv = vals[off[:, j] + 1]
        out = out + ((w * alpha) * vv if sse else (w * vv) * alpha)
    return out, nv


# ---- FilterReg in FP64 -----------------------------------------------------------------------------------------------------
def move(source, rot, t):
    """The source moved in FP64 in a fixed order, no FMA: x' = ((R00 x + R01 y) + R02 z) + t0 (the device loop's order)."""
    s = np.asarray(source, np.float64)
    d = s.shape[1]
    out = np.empty_like(s)
    for a in range(d):
        acc = rot[a, 0] * s[:, 0]
        for b in range(1, d):
            acc = acc + rot[a, b] * s[:, b]
        out[:, a] = acc + t[a]
    return out


def features(t_source, target, sigma2):
    """fin = [t_source / sigma ; target / sigma] rounded once to float32 (filterreg.py:83-88 and pybind11)."""
    sigma = np.sqrt(sigma2)
    return np.r_[np.asarray(t_source, np.float64) / sigma, np.asarray(target, np.float64) / sigma].astype(F)


def expectation_step(t_source, target, sigma2, update_sigma2, target_normals=None, alpha=0.015, impl="ref"):
    """filterreg.py:78-108: (m0, m1, m2, nx, with_blur), float32.  impl "ref": the compiled reference; "numpy": the restatement."""
    filt = ref_filter if impl == "ref" else lattice_filter
    m, d = t_source.shape
    n = target.shape[0]
    fin = features(t_source, target, sigma2)
    blur = True
    size = ref_lattice_size(fin, True) if impl == "ref" else lattice_filter(fin, np.zeros((len(fin), 1)), True)[1]
    if size > n * alpha:
        blur = False
    y = np.asarray(target, np.float64)
    run = lambda v: filt(fin, np.r_[np.zeros((m, v.shape[1])), v], blur)[0][:m]
    m0 = run(np.ones((n, 1))).ravel()
    m1 = run(y)
    m2 = run(np.square(y).sum(axis=1)[:, None]).ravel() if update_sigma2 else None
    nx = run(np.asarray(target_normals, np.float64)) if target_normals is not None else None
    return m0, m1, m2, nx, blur


def kabsch(model, target, weight):
    """cc/kabsch.cc:6-56 in FP64: centres with the weight, H with the weight squared over the sum of weight squared."""
    tw = weight.sum()
    if tw == 0:
        return np.identity(3), np.zeros(3)
    mc, tc = (weight[:, None] * model).sum(0) / tw, (weight[:, None] * target).sum(0) / tw
    w2 = weight * weight
    hh = ((w2[:, None] * (model - mc)).T @ (target - tc)) / w2.sum()
    u, _, vt = np.linalg.svd(hh)
    ss = np.ones(3)
    ss[2] = np.linalg.det(u @ vt.T)                       # det(U V), Eigen's H = U S V^T
    r = vt.T @ np.diag(ss) @ u.T
    return r, tc - r @ mc


def kabsch2d(model, target, weight):
    """cc/kabsch.cc:58-109 in FP64: the rotation angle by atan2 of H."""
    tw = weight.sum()
    if tw == 0:
        return np.identity(2), np.zeros(2)
    mc, tc = (weight[:, None] * model).sum(0) / tw, (weight[:, None] * target).sum(0) / tw
    w2 = weight * weight
    hh = ((w2[:, None] * (model - mc)).T @ (target - tc)) / w2.sum()
    ang = np.arctan2(hh[0, 1] - hh[1, 0], hh[0, 0] + hh[1, 1])
    r = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    return r, tc - r @ mc


def compute_twist_for_pt2pl(model, target, normal, weight):
    """cc/point_to_plane.cc:6-32 in FP64: J^T J and J^T r with the weight, q with the weight squared; the solve of J^T J."""
    res = (normal * (target - model)).sum(1)
    jac = np.c_[np.cross(model, normal), normal]
    ata = (weight[:, None] * jac).T @ jac
    atb = (weight * res) @ jac
    return np.linalg.solve(ata, atb), float((weight * weight * res * res).sum())


def _f32(fn):
    def wrapped(*args):
        out = fn(*[np.asarray(a, F) for a in args])
        return tuple(np.asarray(o, F) if isinstance(o, np.ndarray) else F(o) for o in out)
    return wrapped


# float32 restatements (pybind11 hands the C++ float32 Eigen matrices): the same formulas evaluated on float32 inputs, results float32
kabsch_f32, kabsch2d_f32, pt2pl_f32 = _f32(kabsch), _f32(kabsch2d), _f32(compute_twist_for_pt2pl)


def twist_mul(tw, rot, t):
    """se3_op.twist_mul (se3_op.py:42-53) with twist_trans's exponential map."""
    w, v = tw[:3], tw[3:]
    th = np.linalg.norm(w)
    if th == 0.0:
        tr = np.identity(3)
    else:
        k = w / th
        kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        tr = np.identity(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx
    return tr @ rot, t @ tr.T + v


def maximization_step(t_source, target, estep, rot, t, sigma2, w=0.0, objective_type="pt2pt", target_normals_used=None):
    """filterreg.py:159-196 in FP64.  Returns (rot, t, sigma2, q); q None when no source has m0 != 0."""
    m, dim = t_source.shape
    n = target.shape[0]
    m0, m1, m2, nx = [None if a is None else np.asarray(a, np.float64) for a in estep[:4]]
    c = w / (1.0 - w) * n / m * (2.0 * sigma2 * np.pi) ** (dim / 2.0)
    keep = m0 != 0
    if not keep.any():
        return rot, t, sigma2, None
    m0, m1, ts = m0[keep], m1[keep], t_source[keep]
    m1m0 = (m1.T / m0).T
    m0m0 = m0 / (m0 + c)
    drxdx = np.sqrt(m0m0 * 1.0 / sigma2)
    if objective_type == "pt2pt":
        dr, dt = (kabsch2d if dim == 2 else kabsch)(ts, m1m0, drxdx)
        rx = (drxdx * (ts - m1m0).T).T
        rot, t = dr @ rot, t @ dr.T + dt
        q = np.linalg.norm(rx, ord=2, axis=1).sum()
    elif objective_type == "pt2pl":
        nxm0 = (nx[keep].T / m0).T
        tw, q = compute_twist_for_pt2pl(ts, m1m0, nxm0, drxdx)
        rot, t = twist_mul(tw, rot, t)
    else:
        raise ValueError("Unknown objective_type: %s." % objective_type)
    if m2 is not None:
        m2 = m2[keep]
        sigma2 = ((m0 * np.square(ts).sum(axis=1) - 2.0 * (ts * m1).sum(axis=1) + m2) / (m0 + c)).sum()
        sigma2 /= 3.0 * m0m0.sum()
    return rot, t, sigma2, q


def squared_kernel_sum(x, y):
    """math_utils.squared_kernel_sum (math_utils.py:28-29) in closed form."""
    m, n = x.shape[0], y.shape[0]
    s = n * np.square(x).sum() + m * np.square(y).sum() - 2.0 * x.sum(0) @ y.sum(0)
    return float(s / (m * x.shape[1] * n))


def registration(source, target, target_normals=None, sigma2=None, update_sigma2=False, w=0.0, objective_type="pt2pt", maxiter=50,
                 tol=0.001, min_sigma2=1.0e-4, rot=None, t=None, impl="ref", trace=None):
    """filterreg.py:120-147.  Returns (rot, t, sigma2, q, iterations run); sigma2 is the last M-step's, before the min_sigma2 clamp,
    as the reference's MstepResult holds it."""
    source, target = np.asarray(source, np.float64), np.asarray(target, np.float64)
    dim = source.shape[1]
    rot = np.identity(dim) if rot is None else np.asarray(rot, np.float64)
    t = np.zeros(dim) if t is None else np.asarray(t, np.float64)
    if sigma2 is None:
        sigma2 = max(squared_kernel_sum(source, target), min_sigma2)
    q = None
    res_q = None
    res_s2 = sigma2
    it = 0
    for it in range(1, maxiter + 1):
        ts = move(source, rot, t)
        es = expectation_step(ts, target, sigma2, update_sigma2, target_normals if objective_type == "pt2pl" else None, impl=impl)
        if trace is not None:
            trace.append(es)
        nrot, nt, ns2, res_q = maximization_step(ts, target, es, rot, t, sigma2, w, objective_type)
        if res_q is None:
            res_q = q
            break
        rot, t, sigma2, res_s2 = nrot, nt, max(ns2, min_sigma2), ns2
        if q is not None and abs(res_q - q) < tol:
            break
        q = res_q
    return rot, t, res_s2, res_q, it
