"""ctypes binding of libcpd_b200.so (include/cpd_b200.h).  No torch, no cupy, no CPU fallback:
if the shared library is missing or no CUDA device is visible, using the package raises."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# CPD_B200_LIB: load another build of the same library (tools/tune.sh variants); never a different implementation -- lib() refuses
# anything that exports cpd_is_emulation (the CPU build the test-suite keeps for itself), so the package cannot be given a CPU path this way
LIB_PATH = os.environ.get("CPD_B200_LIB") or os.path.join(_HERE, "libcpd_b200.so")

TF_RIGID, TF_AFFINE, TF_NONRIGID = 0, 1, 2


class CpdParams(ctypes.Structure):
    _fields_ = [("lin", ctypes.c_double * 9), ("t", ctypes.c_double * 3), ("scale", ctypes.c_double),
                ("sigma2", ctypes.c_double), ("q", ctypes.c_double), ("n_p", ctypes.c_double)]


class CpdError(RuntimeError):
    pass


_c_dp = ctypes.POINTER(ctypes.c_double)
_c_fp = ctypes.POINTER(ctypes.c_float)
_PROTOS = {
    "cpd_last_error": (ctypes.c_char_p, []),
    "cpd_version": (ctypes.c_int, []),
    "cpd_device_count": (ctypes.c_int, []),
    "cpd_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "cpd_destroy": (None, [ctypes.c_void_p]),
    "cpd_set_source": (ctypes.c_int, [ctypes.c_void_p, _c_dp, ctypes.c_int64]),
    "cpd_set_target": (ctypes.c_int, [ctypes.c_void_p, _c_dp, ctypes.c_int64, ctypes.c_int64, _c_dp]),
    "cpd_sigma2_init": (ctypes.c_int, [ctypes.c_void_p, _c_dp]),
    "cpd_set_state": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.POINTER(CpdParams)]),
    "cpd_em_step": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(CpdParams)]),
    "cpd_em_run": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.POINTER(CpdParams),
                                  ctypes.POINTER(ctypes.c_int), _c_dp]),
    "cpd_estep": (ctypes.c_int, [ctypes.c_void_p, _c_dp, ctypes.c_double, ctypes.c_double, _c_dp, _c_dp, _c_dp, _c_dp]),
    "cpd_mstep": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, _c_dp, _c_dp, _c_dp, ctypes.c_double,
                                 ctypes.POINTER(CpdParams)]),
    "cpd_bcpd_estep": (ctypes.c_int, [ctypes.c_void_p, _c_dp, ctypes.c_double, _c_dp, _c_dp, ctypes.c_double, ctypes.c_double,
                                      _c_dp, _c_dp, _c_dp, _c_dp]),
    "cpd_last_estep": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp, _c_dp, _c_dp]),
    "cpd_bcpd_begin": (ctypes.c_int, [ctypes.c_void_p, _c_fp, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double]),
    "cpd_bcpd_step": (ctypes.c_int, [ctypes.c_void_p, _c_dp]),
    "cpd_bcpd_get": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(CpdParams), _c_dp, _c_dp, _c_dp, _c_dp]),
    "cpd_bcpd_step_times": (ctypes.c_int, [ctypes.c_void_p, _c_fp]),
    "cpd_bcpd_lowrank_begin": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                              ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_uint64]),
    "cpd_bcpd_lowrank_get": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), _c_dp, _c_dp]),
    "cpd_gmmtree_build": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.POINTER(ctypes.c_int64),
                                         ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "cpd_gmmtree_nodes": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp, _c_dp]),
    "cpd_gmmtree_load": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, _c_dp, _c_dp, _c_dp]),
    "cpd_gmmtree_assign": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32)]),
    "cpd_gmmtree_estep": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp, ctypes.c_double, _c_dp]),
    "cpd_gmmtree_times": (ctypes.c_int, [ctypes.c_void_p, _c_fp, _c_fp]),
    "cpd_nonrigid_begin": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double]),
    "cpd_nonrigid_step": (ctypes.c_int, [ctypes.c_void_p, _c_dp]),
    "cpd_nonrigid_get": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp]),
    "cpd_nonrigid_restart": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double]),
    "cpd_nonrigid_mstep": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp, _c_dp, ctypes.c_double, _c_dp]),
    "cpd_nonrigid_lowrank_begin": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                                  ctypes.c_int, ctypes.c_int, ctypes.c_uint64]),
    "cpd_nonrigid_lowrank_get": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), _c_dp, _c_dp]),
    "cpd_lowrank_gram_product": (ctypes.c_int, [ctypes.c_void_p, _c_dp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_dp]),
    "cpd_nonrigid_set_prior": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_double, _c_dp, _c_dp]),
    "cpd_rbf_kernel": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int,
                                      ctypes.c_double, _c_fp]),
    "cpd_imq_kernel": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int,
                                      ctypes.c_double, _c_fp]),
    "cpd_gauss_transform": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int, ctypes.c_double,
                                           _c_dp, ctypes.c_int, _c_dp]),
    "cpd_gmm_fit": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int64), ctypes.c_double, ctypes.c_double,
                                   ctypes.c_int, _c_dp, _c_dp, _c_dp, ctypes.POINTER(ctypes.c_int), _c_dp]),
    "cpd_l2_dist": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int,
                                   ctypes.c_double, _c_dp, _c_dp]),
    "cpd_tps_kernel": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int, _c_fp]),
    "cpd_ocsvm_fit": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                     ctypes.c_int64, _c_dp, _c_dp, ctypes.POINTER(ctypes.c_int64)]),
    "cpd_lattice_filter": (ctypes.c_int, [ctypes.c_int, _c_fp, ctypes.c_int64, ctypes.c_int, _c_fp, ctypes.c_int, ctypes.c_int, _c_fp,
                                          ctypes.POINTER(ctypes.c_int64)]),
    "cpd_filterreg_estep": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int, _c_dp, ctypes.c_double,
                                           ctypes.c_int, ctypes.c_double, _c_fp, _c_fp, _c_fp, _c_fp, ctypes.POINTER(ctypes.c_int), _c_fp]),
    "cpd_filterreg_begin": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64,
                                           ctypes.c_int, _c_dp, ctypes.c_int, ctypes.c_double]),
    "cpd_filterreg_step": (ctypes.c_int, [ctypes.c_void_p, _c_dp, _c_dp, ctypes.c_double, ctypes.c_double, _c_dp]),
    "cpd_filterreg_get": (ctypes.c_int, [ctypes.c_void_p, _c_fp, _c_fp, _c_fp, _c_fp, ctypes.POINTER(ctypes.c_int),
                                         ctypes.POINTER(ctypes.c_int64), _c_fp]),
    "cpd_filterreg_end": (None, [ctypes.c_void_p]),
    "cpd_batch_register": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_dp, ctypes.POINTER(ctypes.c_int64), _c_dp,
                                          ctypes.POINTER(ctypes.c_int64), ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int,
                                          ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]),
    "cpd_squared_kernel_sum": (ctypes.c_int, [ctypes.c_int, _c_dp, ctypes.c_int64, _c_dp, ctypes.c_int64, ctypes.c_int, _c_dp]),
    "cpd_comm_unique_id": (ctypes.c_int, [ctypes.c_char_p]),
    "cpd_comm_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p]),
    "cpd_comm_destroy": (ctypes.c_int, [ctypes.c_void_p]),
    "cpd_comm_attach": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]),
    "cpd_p2p_local_handle": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p]),
    "cpd_p2p_attach": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]),
    "cpd_plan_work": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                     ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]),
    "cpd_p2p_detach": (ctypes.c_int, [ctypes.c_void_p]),
    "cpd_timer_start": (ctypes.c_int, [ctypes.c_void_p]),
    "cpd_timer_stop": (ctypes.c_int, [ctypes.c_void_p, _c_fp]),
    "cpd_sync": (ctypes.c_int, [ctypes.c_void_p]),
    "cpd_event_record": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "cpd_event_elapsed": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, _c_fp]),
    "cpd_set_profiling": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "cpd_stage_times": (ctypes.c_int, [ctypes.c_void_p, _c_fp]),
    "cpd_lowrank_setup_times": (ctypes.c_int, [ctypes.c_void_p, _c_fp]),
    "cpd_launch_count": (ctypes.c_int64, [ctypes.c_void_p]),
    "cpd_flush_l2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64]),
    "cpd_microbench": (ctypes.c_int, [ctypes.c_int, _c_dp]),
}
EXPORTED = tuple(_PROTOS)
_lib = None


def _load(path):
    """dlopen `path` and attach the prototypes of include/cpd_b200.h."""
    handle = ctypes.CDLL(path)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(handle, name)
        fn.restype = res
        fn.argtypes = args
    return handle


def lib():
    """The loaded shared library (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CpdError("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(or `make -C probreg_b200/csrc`); probreg_b200 has no CPU path" % LIB_PATH)
        loaded = _load(LIB_PATH)
        if hasattr(loaded, "cpd_is_emulation"):
            raise CpdError("%s is the CPU emulation used by the tests (it exports cpd_is_emulation): probreg_b200 has no CPU path "
                           "and will not load it as the product library" % LIB_PATH)
        _lib = loaded
    return _lib


def check(code):
    if code != 0:
        raise CpdError("libcpd_b200: %s (code %d)" % (lib().cpd_last_error().decode(), code))


def as_cloud(a, dim=None):
    """C-order float64 (count x D) view/copy of `a` (what cv() at probreg/cpd.py:444 hands on)."""
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    assert arr.ndim == 2, "source and target must have 2 dimensions."
    if dim is not None and arr.shape[1] != dim:
        raise ValueError("expected %d-D points, got %d-D" % (dim, arr.shape[1]))
    return arr


def dptr(a):
    return a.ctypes.data_as(_c_dp) if a is not None else None


class Handle(object):
    """RAII wrapper of cpd_ctx*: one GPU, one stream."""

    def __init__(self, dim, device=0, stream=None):
        if dim not in (2, 3):
            raise ValueError("probreg_b200 supports 2-D and 3-D points, got %d-D" % dim)
        self._h = ctypes.c_void_p()
        self.dim = dim
        self.device = device
        self._lib = lib()          # a handle is destroyed by the library that created it
        check(self._lib.cpd_create(ctypes.byref(self._h), device, dim, ctypes.c_void_p(stream) if stream else None))
        self.m = 0
        self.n = 0
        self.gmmtree_levels = 0

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.cpd_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- data
    def set_source(self, source):
        src = as_cloud(source, self.dim)
        check(self._lib.cpd_set_source(self._h, dptr(src), src.shape[0]))
        self.m = src.shape[0]

    def set_target(self, target, n_global=None, frame_origin=None):
        tgt = as_cloud(target, self.dim)
        n_global = tgt.shape[0] if n_global is None else int(n_global)
        org = None if frame_origin is None else np.ascontiguousarray(frame_origin, dtype=np.float64)
        check(self._lib.cpd_set_target(self._h, dptr(tgt), tgt.shape[0], n_global, dptr(org)))
        self.n = tgt.shape[0]

    def sigma2_init(self):
        out = ctypes.c_double()
        check(self._lib.cpd_sigma2_init(self._h, ctypes.byref(out)))
        return out.value

    # -- EM
    def set_state(self, tf_kind, update_scale, w, lin, t, scale, sigma2, q):
        p = CpdParams()
        d = self.dim
        lin = np.asarray(lin, dtype=np.float64).reshape(d, d)
        for i in range(d):
            for j in range(d):
                p.lin[i * d + j] = lin[i, j]
        tt = np.asarray(t, dtype=np.float64).reshape(d)
        for i in range(d):
            p.t[i] = tt[i]
        p.scale, p.sigma2, p.q = float(scale), float(sigma2), float(q)
        check(self._lib.cpd_set_state(self._h, tf_kind, int(bool(update_scale)), float(w), ctypes.byref(p)))

    def _unpack(self, p):
        d = self.dim
        lin = np.array(p.lin[: d * d], dtype=np.float64).reshape(d, d)
        t = np.array(p.t[:d], dtype=np.float64)
        return lin, t, p.scale, p.sigma2, p.q, p.n_p

    def em_step(self, read=True):
        if not read:
            check(self._lib.cpd_em_step(self._h, None))
            return None
        p = CpdParams()
        check(self._lib.cpd_em_step(self._h, ctypes.byref(p)))
        return self._unpack(p)

    def em_run(self, maxiter, tol, trace=False):
        p = CpdParams()
        it = ctypes.c_int()
        tr = np.zeros((max(maxiter, 1), 2)) if trace else None
        check(self._lib.cpd_em_run(self._h, int(maxiter), float(tol), ctypes.byref(p), ctypes.byref(it), dptr(tr)))
        out = self._unpack(p) + (it.value,)
        return out + (tr[: it.value],) if trace else out

    def estep(self, t_source, sigma2, w, want_pt1=True, want_p1=True, want_px=True):
        ts = as_cloud(t_source, self.dim)
        if ts.shape[0] != self.m:
            raise ValueError("t_source has %d rows, the handle's source has %d" % (ts.shape[0], self.m))
        pt1 = np.empty(self.n) if want_pt1 else None
        p1 = np.empty(self.m) if want_p1 else None
        px = np.empty((self.m, self.dim)) if want_px else None
        n_p = ctypes.c_double()
        check(self._lib.cpd_estep(self._h, dptr(ts), float(sigma2), float(w), dptr(pt1), dptr(p1), dptr(px), ctypes.byref(n_p)))
        return pt1, p1, px, n_p.value

    def bcpd_estep(self, t_source, scale, alpha, sigma_diag, sigma2, w):
        """(nu_d, nu, px, n_p) of probreg/bcpd.py:53-72 for the handle's target."""
        ts = as_cloud(t_source, self.dim)
        al = np.ascontiguousarray(alpha, dtype=np.float64)
        sd = np.ascontiguousarray(sigma_diag, dtype=np.float64)
        if ts.shape[0] != self.m or al.shape != (self.m,) or sd.shape != (self.m,):
            raise ValueError("t_source / alpha / sigma_diag do not match the handle's source count %d" % self.m)
        nu_d, nu, px = np.empty(self.n), np.empty(self.m), np.empty((self.m, self.dim))
        n_p = ctypes.c_double()
        check(self._lib.cpd_bcpd_estep(self._h, dptr(ts), float(scale), dptr(al), dptr(sd), float(sigma2), float(w), dptr(nu_d), dptr(nu),
                                   dptr(px), ctypes.byref(n_p)))
        return nu_d, nu, px, n_p.value

    # -- BCPD registration loop (G^-1, A and Sigma resident on the device)
    def bcpd_begin(self, gmat_inv, lmd, k, sigma2, w):
        """Start CombinedBCPD's loop from the reference's _initialize; gmat_inv: the (m, m) C-contiguous float32 inverse of the
        kernel matrix, in the caller's point order (set_source / set_target first)."""
        if not isinstance(gmat_inv, np.ndarray) or gmat_inv.dtype != np.float32:
            raise ValueError("gmat_inv must be a float32 numpy array, got %s" % getattr(gmat_inv, "dtype", type(gmat_inv)))
        if gmat_inv.shape != (self.m, self.m):
            raise ValueError("gmat_inv must be %d x %d (the handle's source count), got %s" % (self.m, self.m, gmat_inv.shape))
        if not gmat_inv.flags["C_CONTIGUOUS"]:
            raise ValueError("gmat_inv must be C-contiguous (row-major)")
        check(self._lib.cpd_bcpd_begin(self._h, gmat_inv.ctypes.data_as(_c_fp), float(lmd), float(k), float(sigma2), float(w)))

    def bcpd_lowrank_begin(self, c, lmd, k, sigma2, w, rank, power_iters=2, seed=0):
        """Start CombinedBCPD's loop with the IMQ kernel matrix (parameter c) replaced by a rank-`rank` factorisation built on the
        device (set_source / set_target first); bcpd_step / bcpd_get then run the low-rank loop."""
        for name, val in (("rank", rank), ("power_iters", power_iters), ("seed", seed)):
            if isinstance(val, bool) or not isinstance(val, (int, np.integer)):
                raise ValueError("%s must be an integer, got %r" % (name, val))
        if not 1 <= rank <= 1024:
            raise ValueError("rank must be in 1..1024, got %d" % rank)
        if not 0 <= power_iters <= 8:
            raise ValueError("power_iters must be in 0..8, got %d" % power_iters)
        if not (np.isfinite(c) and c > 0):
            raise ValueError("c must be a positive finite number, got %r" % (c,))
        check(self._lib.cpd_bcpd_lowrank_begin(self._h, float(c), float(lmd), float(k), float(sigma2), float(w), int(rank), int(power_iters),
                                               int(seed)))

    def bcpd_lowrank_factors(self):
        """(Q (m x rank), Bc (rank x rank)) of the low-rank BCPD loop: G ~= Q Bc Q^T, Q in the caller's point order."""
        k = ctypes.c_int()
        check(self._lib.cpd_bcpd_lowrank_get(self._h, ctypes.byref(k), None, None))
        q, b = np.empty((self.m, k.value)), np.empty((k.value, k.value))
        check(self._lib.cpd_bcpd_lowrank_get(self._h, None, dptr(q), dptr(b)))
        return q, b

    def bcpd_step(self):
        """One iteration; returns the new sigma2."""
        out = ctypes.c_double()
        check(self._lib.cpd_bcpd_step(self._h, ctypes.byref(out)))
        return out.value

    def bcpd_get(self, v=True, moved=False, alpha=False, sigma_diag=False):
        """(rot, t, scale, sigma2, v, moved, alpha, sigma_diag) of the loop's current state in the caller's order; the arrays not
        asked for are None."""
        p = CpdParams()
        va = np.empty((self.m, self.dim)) if v else None
        mv = np.empty((self.m, self.dim)) if moved else None
        al = np.empty(self.m) if alpha else None
        sd = np.empty(self.m) if sigma_diag else None
        check(self._lib.cpd_bcpd_get(self._h, ctypes.byref(p), dptr(va), dptr(mv), dptr(al), dptr(sd)))
        rot, t, scale, sigma2 = self._unpack(p)[:4]
        return rot, t, scale, sigma2, va, mv, al, sd

    def bcpd_step_times(self):
        ms = (ctypes.c_float * 5)()
        check(self._lib.cpd_bcpd_step_times(self._h, ms))
        return {"estep_ms": ms[0], "system_ms": ms[1], "getrf_ms": ms[2], "getrs_ms": ms[3], "rest_ms": ms[4]}

    def last_estep(self):
        pt1, p1, px = np.empty(self.n), np.empty(self.m), np.empty((self.m, self.dim))
        n_p = ctypes.c_double()
        check(self._lib.cpd_last_estep(self._h, dptr(pt1), dptr(p1), dptr(px), ctypes.byref(n_p)))
        return pt1, p1, px, n_p.value

    def mstep(self, tf_kind, update_scale, pt1, p1, px, n_p):
        pt1 = np.ascontiguousarray(pt1, dtype=np.float64)
        p1 = np.ascontiguousarray(p1, dtype=np.float64)
        px = as_cloud(px, self.dim)
        if pt1.shape[0] != self.n or p1.shape[0] != self.m or px.shape[0] != self.m:
            raise ValueError("EstepResult shapes do not match the handle's source/target")
        p = CpdParams()
        check(self._lib.cpd_mstep(self._h, tf_kind, int(bool(update_scale)), dptr(pt1), dptr(p1), dptr(px), float(n_p),
                              ctypes.byref(p)))
        return self._unpack(p)

    # -- GMMTree (3-D handles only)
    @staticmethod
    def gmmtree_total(tree_level):
        """number of nodes of a tree of `tree_level` levels: 8 (8^L - 1) / 7"""
        return 8 * (8 ** tree_level - 1) // 7

    def gmmtree_build(self, tree_level, lambda_s, lambda_d, leaf_seeds, maxiter=1000):
        """buildGmmTree on the handle's source from the 8^L leaf seeds (point indices, caller's order); returns the iterations
        each level ran."""
        seeds = np.ascontiguousarray(leaf_seeds, dtype=np.int64)
        if not 1 <= int(tree_level) <= 5:
            raise ValueError("tree_level must be in 1..5, got %r" % (tree_level,))
        if seeds.shape != (8 ** int(tree_level),):
            raise ValueError("leaf_seeds must hold 8^tree_level = %d indices, got shape %s" % (8 ** int(tree_level), seeds.shape))
        iters = np.zeros(int(tree_level), dtype=np.int32)
        check(self._lib.cpd_gmmtree_build(self._h, int(tree_level), float(lambda_s), float(lambda_d),
                                          seeds.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), int(maxiter),
                                          iters.ctypes.data_as(ctypes.POINTER(ctypes.c_int))))
        self.gmmtree_levels = int(tree_level)
        return iters

    def gmmtree_nodes(self):
        """(pi (n_total,), mu (n_total, 3), cov (n_total, 3, 3)) of the handle's tree"""
        total = self.gmmtree_total(self.gmmtree_levels)
        pi, mu, cov = np.empty(total), np.empty((total, 3)), np.empty((total, 3, 3))
        check(self._lib.cpd_gmmtree_nodes(self._h, dptr(pi), dptr(mu), dptr(cov)))
        return pi, mu, cov

    def gmmtree_load(self, tree_level, pi, mu, cov):
        total = self.gmmtree_total(int(tree_level)) if 1 <= int(tree_level) <= 5 else 0
        pi = np.ascontiguousarray(pi, dtype=np.float64)
        mu = np.ascontiguousarray(mu, dtype=np.float64)
        cov = np.ascontiguousarray(cov, dtype=np.float64)
        if total and (pi.shape != (total,) or mu.shape != (total, 3) or cov.shape != (total, 3, 3)):
            raise ValueError("a tree of %d levels has %d nodes: pi (n,), mu (n, 3), cov (n, 3, 3)" % (tree_level, total))
        check(self._lib.cpd_gmmtree_load(self._h, int(tree_level), dptr(pi), dptr(mu), dptr(cov)))
        self.gmmtree_levels = int(tree_level)

    def gmmtree_assign(self):
        """the node each source point was assigned to in the last E-step of the build (caller's order)"""
        out = np.empty(self.m, dtype=np.int32)
        check(self._lib.cpd_gmmtree_assign(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))
        return out

    def gmmtree_estep(self, rot, t, lambda_c):
        """moments (n_total, 13) -- m0, m1 (3), m2 (3 x 3) -- of the handle's target moved by rot x + t"""
        r = np.ascontiguousarray(rot, dtype=np.float64).reshape(9)
        tt = np.ascontiguousarray(t, dtype=np.float64).reshape(3)
        out = np.empty((self.gmmtree_total(self.gmmtree_levels), 13))
        check(self._lib.cpd_gmmtree_estep(self._h, dptr(r), dptr(tt), float(lambda_c), dptr(out)))
        return out

    def gmmtree_times(self):
        lv, es = (ctypes.c_float * 5)(), ctypes.c_float()
        check(self._lib.cpd_gmmtree_times(self._h, lv, ctypes.byref(es)))
        return {"level_ms": list(lv), "estep_ms": es.value}

    # -- GMMReg: the spherical GMM fit of the source
    def gmm_fit(self, n_components, seeds, reg_covar=1e-6, tol=1e-3, max_iter=100):
        """features.GMM's spherical GaussianMixture fit of the handle's source from one-hot responsibilities at `seeds` (distinct
        point indices, caller's order); returns (weights (K,), means (K, D), variances (K,), n_iter, lower bound per iteration)."""
        sd = np.ascontiguousarray(seeds, dtype=np.int64)
        k = int(n_components)
        if sd.shape != (k,):
            raise ValueError("seeds must hold n_components = %d indices, got shape %s" % (k, sd.shape))
        w, mu, var = np.empty(k), np.empty((k, self.dim)), np.empty(k)
        lb = np.empty(max(int(max_iter), 1))
        it = ctypes.c_int()
        check(self._lib.cpd_gmm_fit(self._h, k, sd.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), float(reg_covar), float(tol),
                                    int(max_iter), dptr(w), dptr(mu), dptr(var), ctypes.byref(it), dptr(lb)))
        return w, mu, var, it.value, lb[: it.value]

    # -- non-rigid (dense G on the device)
    def nonrigid_begin(self, beta, lmd, sigma2, w):
        check(self._lib.cpd_nonrigid_begin(self._h, float(beta), float(lmd), float(sigma2), float(w)))

    def nonrigid_lowrank_begin(self, beta, lmd, sigma2, w, rank, power_iters=2, seed=0):
        check(self._lib.cpd_nonrigid_lowrank_begin(self._h, float(beta), float(lmd), float(sigma2), float(w), int(rank), int(power_iters),
                                               int(seed)))

    def nonrigid_lowrank_factors(self):
        """(Q (m x rank), Bc (rank x rank)) with G ~= Q Bc Q^T, Q in the caller's point order."""
        k = ctypes.c_int()
        check(self._lib.cpd_nonrigid_lowrank_get(self._h, ctypes.byref(k), None, None))
        q, b = np.empty((self.m, k.value)), np.empty((k.value, k.value))
        check(self._lib.cpd_nonrigid_lowrank_get(self._h, None, dptr(q), dptr(b)))
        return q, b

    GRAM_TENSOR_CORES, GRAM_CUDA_CORES = 0, 1

    def lowrank_gram_product(self, x, kernel, world=1, rank=0):
        """G x (m x cols) for the G of the last low-rank set-up (nonrigid_lowrank_begin: Gaussian, bcpd_lowrank_begin: inverse
        multiquadric), by one kernel (GRAM_TENSOR_CORES or GRAM_CUDA_CORES);
        with world > 1 only the rows of `rank`'s share are filled.  A test / diagnostic entry: the factors stay as they were."""
        xa = np.ascontiguousarray(x, dtype=np.float64)
        if xa.ndim != 2 or xa.shape[0] != self.m:
            raise ValueError("x must be m x cols with m = %d, got %s" % (self.m, xa.shape))
        out = np.empty_like(xa)
        check(self._lib.cpd_lowrank_gram_product(self._h, dptr(xa), xa.shape[1], int(kernel), int(world), int(rank), dptr(out)))
        return out

    def nonrigid_set_prior(self, alpha, p1_tilde, px_tilde):
        if p1_tilde is None:
            check(self._lib.cpd_nonrigid_set_prior(self._h, 1.0, None, None))
            return
        p1t = np.ascontiguousarray(p1_tilde, dtype=np.float64)
        pxt = as_cloud(px_tilde, self.dim)
        if p1t.shape != (self.m,) or pxt.shape[0] != self.m:
            raise ValueError("prior shapes do not match the handle's source")
        check(self._lib.cpd_nonrigid_set_prior(self._h, float(alpha), dptr(p1t), dptr(pxt)))

    def nonrigid_moved(self):
        t = np.empty((self.m, self.dim))
        check(self._lib.cpd_nonrigid_get(self._h, None, dptr(t)))
        return t

    def nonrigid_restart(self, lmd, sigma2, w):
        check(self._lib.cpd_nonrigid_restart(self._h, float(lmd), float(sigma2), float(w)))

    def nonrigid_mstep(self, pt1, p1, px, sigma2_p):
        pt1 = np.ascontiguousarray(pt1, dtype=np.float64)
        p1 = np.ascontiguousarray(p1, dtype=np.float64)
        px = as_cloud(px, self.dim)
        if pt1.shape[0] != self.n or p1.shape[0] != self.m or px.shape[0] != self.m:
            raise ValueError("EstepResult shapes do not match the handle's source/target")
        out = ctypes.c_double()
        check(self._lib.cpd_nonrigid_mstep(self._h, dptr(pt1), dptr(p1), dptr(px), float(sigma2_p), ctypes.byref(out)))
        return out.value

    def nonrigid_step(self):
        out = ctypes.c_double()
        check(self._lib.cpd_nonrigid_step(self._h, ctypes.byref(out)))
        return out.value

    def nonrigid_w(self):
        w = np.empty((self.m, self.dim))
        check(self._lib.cpd_nonrigid_get(self._h, dptr(w), None))
        return w

    # -- multi-GPU
    def attach_comm(self, nccl_comm, world_size, rank):
        """nccl_comm: the value returned by comm_create (borrowed; it must outlive the handle)."""
        check(self._lib.cpd_comm_attach(self._h, nccl_comm, world_size, rank))

    def p2p_local_handle(self):
        buf = ctypes.create_string_buffer(64)
        check(self._lib.cpd_p2p_local_handle(self._h, buf))
        return buf.raw

    def p2p_attach(self, handles, world_size, rank):
        blob = b"".join(handles)
        assert len(blob) == 64 * world_size
        check(self._lib.cpd_p2p_attach(self._h, blob, world_size, rank))

    def p2p_detach(self):
        check(self._lib.cpd_p2p_detach(self._h))

    # -- measurement
    def timer_start(self):
        check(self._lib.cpd_timer_start(self._h))

    def timer_stop(self):
        ms = ctypes.c_float()
        check(self._lib.cpd_timer_stop(self._h, ctypes.byref(ms)))
        return ms.value

    def sync(self):
        check(self._lib.cpd_sync(self._h))

    def event_record(self, idx):
        check(self._lib.cpd_event_record(self._h, idx))

    def event_elapsed(self, a, b):
        ms = ctypes.c_float()
        check(self._lib.cpd_event_elapsed(self._h, a, b, ctypes.byref(ms)))
        return ms.value

    def set_profiling(self, on):
        check(self._lib.cpd_set_profiling(self._h, int(on)))

    def stage_times(self):
        ms = (ctypes.c_float * 6)()
        check(self._lib.cpd_stage_times(self._h, ms))
        return list(ms)

    def lowrank_setup_times(self):
        ms = (ctypes.c_float * 3)()
        check(self._lib.cpd_lowrank_setup_times(self._h, ms))
        return {"gram_products_ms": ms[0], "orthonormalisation_ms": ms[1], "core_ms": ms[2]}

    def launch_count(self):
        return int(lib().cpd_launch_count(self._h))

    def flush_l2(self, nbytes=0):
        check(self._lib.cpd_flush_l2(self._h, nbytes))


def unique_id():
    buf = ctypes.create_string_buffer(128)
    check(lib().cpd_comm_unique_id(buf))
    return buf.raw


def plan_work(ntiles, nunits, slots, last_tile_cost=1.0):
    """(items (k x 4 int array: tile, first unit, end unit, slot), max partial slots per tile) -- host only."""
    n, mx = ctypes.c_int(), ctypes.c_int()
    check(lib().cpd_plan_work(ntiles, nunits, slots, float(last_tile_cost), None, 0, ctypes.byref(n), ctypes.byref(mx)))
    buf = np.zeros((n.value, 4), dtype=np.int32)
    check(lib().cpd_plan_work(ntiles, nunits, slots, float(last_tile_cost), buf.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), n.value,
                              ctypes.byref(n), ctypes.byref(mx)))
    return buf, mx.value


def l2_dist(mu_source, phi_source, mu_target, phi_target, sigma, device=0):
    """(f, g) of cost_functions.compute_l2_dist by direct FP64 sums on the device (cpd_l2_dist); g: (n_source, D)."""
    ms, mt = as_cloud(mu_source), as_cloud(mu_target)
    ps, pt = np.ascontiguousarray(phi_source, dtype=np.float64), np.ascontiguousarray(phi_target, dtype=np.float64)
    if ms.shape[1] != mt.shape[1] or ps.shape != (ms.shape[0],) or pt.shape != (mt.shape[0],):
        raise ValueError("mixture shapes do not match: means %s / %s, weights %s / %s" % (ms.shape, mt.shape, ps.shape, pt.shape))
    f = ctypes.c_double()
    g = np.empty(ms.shape)
    check(lib().cpd_l2_dist(device, dptr(ms), ms.shape[0], dptr(ps), dptr(mt), mt.shape[0], dptr(pt), ms.shape[1], float(sigma),
                            ctypes.byref(f), dptr(g)))
    return f.value, g


def ocsvm_fit(x, nu, gamma, tol=1e-3, max_iter=None, device=0):
    """(alpha (every point), rho, n_iter) of sklearn's OneClassSVM(kernel="rbf", nu, gamma, tol).fit on the device (cpd_ocsvm_fit);
    max_iter None: libsvm's cap max(10^7, 100 n)."""
    xa = as_cloud(x)
    n = xa.shape[0]
    max_iter = max(10_000_000, 100 * n) if max_iter is None else int(max_iter)
    alpha = np.empty(n)
    rho, it = ctypes.c_double(), ctypes.c_int64()
    check(lib().cpd_ocsvm_fit(device, dptr(xa), n, xa.shape[1], float(nu), float(gamma), float(tol), max_iter, dptr(alpha),
                              ctypes.byref(rho), ctypes.byref(it)))
    return alpha, rho.value, it.value


def batch_register(src, src_off, tgt, tgt_off, dim, tf_kind, update_scale, w, maxiter, tol, init=None, device=0):
    """Many rigid / affine registrations in one call (cpd_batch_register).  src, tgt: the concatenated clouds (rows x dim);
    src_off, tgt_off: the B + 1 row offsets of the pairs; init: None or B (lin (dim x dim), t (dim), scale) tuples.
    Returns a list of B (lin, t, scale, sigma2, q, n_p) tuples and the iterations each pair ran (int array)."""
    s, t = as_cloud(src, dim), as_cloud(tgt, dim)
    so = np.ascontiguousarray(src_off, dtype=np.int64)
    to = np.ascontiguousarray(tgt_off, dtype=np.int64)
    b = so.shape[0] - 1
    if b < 1 or to.shape != so.shape:
        raise ValueError("src_off and tgt_off must both hold B + 1 >= 2 offsets, got %s and %s" % (so.shape, to.shape))
    ini = None
    if init is not None:
        ini = (CpdParams * b)()
        for k, (lin, tt, scale) in enumerate(init):
            lin = np.asarray(lin, dtype=np.float64).reshape(dim, dim)
            tt = np.asarray(tt, dtype=np.float64).reshape(dim)
            for i in range(dim):
                ini[k].t[i] = tt[i]
                for j in range(dim):
                    ini[k].lin[i * dim + j] = lin[i, j]
            ini[k].scale = float(scale)
    out = (CpdParams * b)()
    iters = np.zeros(b, dtype=np.int32)
    check(lib().cpd_batch_register(int(device), int(dim), b, dptr(s), so.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), dptr(t),
                                   to.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), int(tf_kind), int(bool(update_scale)), float(w),
                                   int(maxiter), float(tol), ctypes.cast(ini, ctypes.c_void_p) if ini is not None else None,
                                   ctypes.cast(out, ctypes.c_void_p), iters.ctypes.data_as(ctypes.POINTER(ctypes.c_int))))
    res = []
    for k in range(b):
        p = out[k]
        res.append((np.array(p.lin[: dim * dim], dtype=np.float64).reshape(dim, dim), np.array(p.t[:dim], dtype=np.float64), p.scale,
                    p.sigma2, p.q, p.n_p))
    return res, iters


def fptr(a):
    return None if a is None else a.ctypes.data_as(_c_fp)


def lattice_filter(feature, values=None, with_blur=True, device=0):
    """(filtered values (n x vs float32) or None, lattice size) of the reference's permutohedral lattice (cpd_lattice_filter):
    Permutohedral(feature, with_blur).filter(values) with feature and values rounded to float32 as pybind11 rounds them."""
    f = np.ascontiguousarray(feature, dtype=np.float32)
    if f.ndim != 2:
        raise ValueError("feature must be (n x d), got shape %s" % (f.shape,))
    n, d = f.shape
    size = ctypes.c_int64()
    if values is None:
        check(lib().cpd_lattice_filter(device, fptr(f), n, d, None, 0, int(bool(with_blur)), None, ctypes.byref(size)))
        return None, size.value
    v = np.ascontiguousarray(values, dtype=np.float32)
    if v.ndim == 1:
        v = v[:, None]
    if v.ndim != 2 or v.shape[0] != n:
        raise ValueError("values must have one row per feature point: %s for %d points" % (v.shape, n))
    out = np.empty_like(v)
    check(lib().cpd_lattice_filter(device, fptr(f), n, d, fptr(v), v.shape[1], int(bool(with_blur)), fptr(out), ctypes.byref(size)))
    return out, size.value


def filterreg_estep(t_source, target, sigma2, update_sigma2, target_normals=None, alpha=0.015, device=0, stage_ms=None):
    """(m0, m1, m2 or None, nx or None, with_blur) of FilterReg.expectation_step on the device (cpd_filterreg_estep), float32."""
    s, t = as_cloud(t_source), as_cloud(target)
    m, d = s.shape
    n = t.shape[0]
    if t.shape[1] != d:
        raise ValueError("source and target must have the same dimension: %d and %d" % (d, t.shape[1]))
    nrm = None if target_normals is None else as_cloud(target_normals, d)
    if nrm is not None and nrm.shape[0] != n:
        raise ValueError("target_normals must have one row per target point: %d for %d" % (nrm.shape[0], n))
    m0, m1 = np.empty(m, np.float32), np.empty((m, d), np.float32)
    m2 = np.empty(m, np.float32) if update_sigma2 else None
    nx = np.empty((m, d), np.float32) if nrm is not None else None
    blur = ctypes.c_int()
    check(lib().cpd_filterreg_estep(device, dptr(s), m, dptr(t), n, d, dptr(nrm) if nrm is not None else None, float(sigma2),
                                    int(bool(update_sigma2)), float(alpha), fptr(m0), fptr(m1), fptr(m2), fptr(nx), ctypes.byref(blur),
                                    fptr(stage_ms)))
    return m0, m1, m2, nx, bool(blur.value)


class FilterRegLoop(object):
    """The FilterReg loop's device state (cpd_filterreg_begin / step / get / end): the clouds uploaded once; step() moves the
    source, runs the E-step and returns the 49 FP64 M-step sums of include/cpd_b200.h."""
    N_MOMENTS = 49

    def __init__(self, source, target, target_normals=None, update_sigma2=False, alpha=0.015, device=0):
        s, t = as_cloud(source), as_cloud(target)
        if t.shape[1] != s.shape[1]:
            raise ValueError("source and target must have the same dimension: %d and %d" % (s.shape[1], t.shape[1]))
        nrm = None if target_normals is None else as_cloud(target_normals, s.shape[1])
        if nrm is not None and nrm.shape[0] != t.shape[0]:
            raise ValueError("target_normals must have one row per target point: %d for %d" % (nrm.shape[0], t.shape[0]))
        self.m, self.d = s.shape
        self.update_sigma2, self.has_normals = bool(update_sigma2), nrm is not None
        self._lib = lib()
        h = ctypes.c_void_p()
        check(self._lib.cpd_filterreg_begin(ctypes.byref(h), device, dptr(s), self.m, dptr(t), t.shape[0], self.d, dptr(nrm),
                                            int(self.update_sigma2), float(alpha)))
        self._h = h

    def step(self, rot, t, sigma2, w):
        mom = np.empty(self.N_MOMENTS)
        r = np.ascontiguousarray(rot, np.float64)
        tt = np.ascontiguousarray(t, np.float64)
        check(self._lib.cpd_filterreg_step(self._h, dptr(r), dptr(tt), float(sigma2), float(w), dptr(mom)))
        return mom

    def last_estep(self):
        """(m0, m1, m2 or None, nx or None, with_blur) of the last step's E-step."""
        m, d = self.m, self.d
        m0, m1 = np.empty(m, np.float32), np.empty((m, d), np.float32)
        m2 = np.empty(m, np.float32) if self.update_sigma2 else None
        nx = np.empty((m, d), np.float32) if self.has_normals else None
        blur = ctypes.c_int()
        check(self._lib.cpd_filterreg_get(self._h, fptr(m0), fptr(m1), fptr(m2), fptr(nx), ctypes.byref(blur), None, None))
        return m0, m1, m2, nx, bool(blur.value)

    def device_bytes(self):
        b = ctypes.c_int64()
        check(self._lib.cpd_filterreg_get(self._h, None, None, None, None, None, ctypes.byref(b), None))
        return b.value

    def stage_ms(self):
        ms = np.zeros(6, np.float32)
        check(self._lib.cpd_filterreg_get(self._h, None, None, None, None, None, None, fptr(ms)))
        return ms

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self._lib.cpd_filterreg_end(h)
            self._h = None


def comm_create(device, world_size, rank, uid):
    """Collective: every rank calls it once with the same unique id.  Returns an opaque pointer."""
    c = ctypes.c_void_p()
    check(lib().cpd_comm_create(ctypes.byref(c), device, world_size, rank, uid))
    return c


def comm_destroy(c):
    check(lib().cpd_comm_destroy(c))


def microbench(device=0):
    out = (ctypes.c_double * 9)()
    check(lib().cpd_microbench(device, out))
    return {"ffma_tflops": out[0], "mufu_ex2_gops": out[1], "sm_mhz": out[2], "sm_count": int(out[3]),
            "ffma2_tflops": out[4], "mix_11p1_gpairs": out[5], "mix_packed_gpairs": out[6], "mix_7p1_gpairs": out[7], "ffma2_plus_ffma_tflops": out[8]}
