"""Coherent Point Drift on one or more B200s -- the API surface of ``probreg.cpd``.

Drop-in for probreg/cpd.py: ``registration_cpd``, ``RigidCPD``, ``AffineCPD``, ``NonRigidCPD``, ``ConstrainedNonRigidCPD``,
``EstepResult``, ``MstepResult`` keep their names, arguments, return types and error behaviour.
What differs is where the work happens: every E-step / M-step runs in hand-written sm_90a
kernels behind the C ABI of ``libcpd_b200.so`` (include/cpd_b200.h).  There is no numpy path
and no CPU fallback; ``use_cuda`` is accepted for signature compatibility and ignored (the
reference's False default would select its numpy path, which does not exist here).

Extensions over the reference signature (all optional, keyword-only in spirit):
``device`` (CUDA ordinal) and ``comm`` (a ``probreg_b200.dist.Communicator``: the target is
sharded over the ranks, one NCCL all-reduce per EM iteration).
"""
import abc
import logging
from collections import namedtuple

import numpy as np

from . import _cabi
from . import transformation as tf
from .log import log

EstepResult = namedtuple("EstepResult", ["pt1", "p1", "px", "n_p"])
MstepResult = namedtuple("MstepResult", ["transformation", "sigma2", "q"])
MstepResult.__doc__ = """Outcome of one M-step (field names as in probreg/cpd.py:18-25).

    transformation -- the current source->target Transformation (host-side value object)
    sigma2         -- isotropic variance of the GMM components
    q              -- objective value used by the convergence test of ``registration``
"""

try:  # optional: accept open3d point clouds like probreg/cpd.py:444 does
    import open3d as _o3

    _PointCloud = _o3.geometry.PointCloud
except Exception:  # pragma: no cover
    class _PointCloud(object):
        pass


def _points(x):
    return np.asarray(x.points if isinstance(x, _PointCloud) else x)


class CoherentPointDrift(abc.ABC):
    """EM driver (probreg/cpd.py:28-120).  The E-step is implemented here, the M-step in the
    subclasses -- both as calls into the CUDA library.

    ``source``: (M, D) array or None; ``use_cuda``: ignored, the sm_90a kernels are the only implementation;
    ``device``: CUDA ordinal (default: the communicator's, else 0); ``comm``: a probreg_b200.dist.Communicator
    for multi-GPU target sharding.
    """

    def __init__(self, source=None, use_cuda=False, device=None, comm=None):
        self._source = None if source is None else _points(source)
        self._tf_type = None
        self._callbacks = []
        self.xp = np
        self._comm = comm
        self._device = (comm.device if comm is not None else 0) if device is None else device
        self._em = None          # handle used by registration()/maximization_step (source = self._source)
        self._es = None          # handle used by stand-alone expectation_step (source = t_source)

    # -- reference API ------------------------------------------------------------------------
    def set_source(self, source):
        self._source = _points(source)

    def set_callbacks(self, callbacks):
        self._callbacks.extend(callbacks)

    @abc.abstractmethod
    def _initialize(self, target):
        return MstepResult(None, None, None)

    def expectation_step(self, t_source, target, sigma2, w=0.0):
        """Expectation step for CPD (probreg/cpd.py:71-88) on the device.

        Host arrays in, host arrays out; P is never materialised.  With a communicator,
        ``target`` is the full cloud, each rank evaluates its shard and ``pt1`` is returned for
        the local shard only while ``p1``/``px``/``n_p`` are the all-reduced global sums.
        """
        t_source, target = np.asarray(t_source), np.asarray(target)
        assert t_source.ndim == 2 and target.ndim == 2, "source and target must have 2 dimensions."
        dim = t_source.shape[1]
        if self._es is None or self._es.dim != dim:
            self._es = self._new_handle(dim)
        self._es.set_source(t_source)
        self._set_target(self._es, target)
        pt1, p1, px, n_p = self._es.estep(t_source, sigma2, w)
        return EstepResult(pt1, p1, px, n_p)

    def maximization_step(self, target, estep_res, sigma2_p=None):
        return self._maximization_step(self._source, target, estep_res, sigma2_p, xp=self.xp)

    @staticmethod
    @abc.abstractmethod
    def _maximization_step(source, target, estep_res, sigma2_p=None, xp=np):
        return None

    def registration(self, target, w=0.0, maxiter=50, tol=0.001):
        """The EM loop of probreg/cpd.py:106-120, resident on the GPU.

        Source and target are uploaded once; each iteration is a fixed sequence of kernel
        launches (transform+pack, E-step pass 1/2, moments, M-step) and the only per-iteration
        host traffic is the 16-double MstepResult needed for callbacks / the ``tol`` test.
        """
        assert not self._tf_type is None, "transformation type is None."
        target = _points(target)
        res = self._initialize(target)      # uploads source/target, sigma2_0 from the device
        h = self._em
        self._push_state(h, res, w)
        q = res.q
        per_iter = bool(self._callbacks) or log.isEnabledFor(logging.DEBUG)
        if not per_iter:
            out = h.em_run(maxiter, tol)
            return self._result_from(out[:6]) if out[6] > 0 else res
        for i in range(maxiter):
            res = self._result_from(h.em_step())
            for c in self._callbacks:
                c(res.transformation)
            log.debug("Iteration: {}, Criteria: {}".format(i, res.q))
            if abs(res.q - q) < tol:
                break
            q = res.q
        return res

    # -- plumbing -----------------------------------------------------------------------------
    def _new_handle(self, dim):
        h = _cabi.Handle(dim, device=self._device)
        if self._comm is not None:
            self._comm.attach(h)
        return h

    def _set_target(self, h, target):
        if self._comm is not None and self._comm.world_size > 1:
            lo, hi = self._comm.shard_bounds(target.shape[0])
            h.set_target(target[lo:hi], n_global=target.shape[0], frame_origin=self._comm.frame_origin(target))
        else:
            h.set_target(target)

    def _em_handle(self, target):
        assert self._source is not None, "source is None."
        dim = self._source.shape[1]
        if self._em is None or self._em.dim != dim:
            self._em = self._new_handle(dim)
        self._em.set_source(self._source)      # always re-uploaded: the caller may have edited it in place
        self._set_target(self._em, target)
        return self._em

    def _squared_kernel_sum(self, source, target):
        # math_utils.squared_kernel_sum (math_utils.py:28-29) on the handle's resident clouds
        return self._em_handle(_points(target)).sigma2_init()

    @abc.abstractmethod
    def _push_state(self, h, res, w):
        pass

    @abc.abstractmethod
    def _result_from(self, out):
        pass


class RigidCPD(CoherentPointDrift):
    """Rigid (rotation + translation, optionally isotropic scale) CPD -- probreg/cpd.py:123-192.

    ``source``: (M, D) array or None (set later with ``set_source``); ``update_scale``: estimate the scale
    (True, default) or keep it at 1; ``tf_init_params``: warm start, keys ``rot``/``t``/``scale``;
    ``use_cuda``: accepted, ignored (module docstring); ``device``/``comm``: see CoherentPointDrift.
    """

    def __init__(self, source=None, update_scale=True, tf_init_params=None, use_cuda=False, device=None, comm=None):
        super(RigidCPD, self).__init__(source, use_cuda, device, comm)
        self._tf_type = tf.RigidTransformation
        self._update_scale = update_scale
        self._tf_init_params = dict(tf_init_params) if tf_init_params else {}

    def _initialize(self, target):
        dim = self._source.shape[1]
        sigma2 = self._squared_kernel_sum(self._source, target)
        q = 1.0 + target.shape[0] * dim * 0.5 * np.log(sigma2)
        params = dict(self._tf_init_params)
        if len(params) == 0:
            params = {"rot": np.identity(dim), "t": np.zeros(dim)}
        params.setdefault("xp", np)
        return MstepResult(self._tf_type(**params), sigma2, q)

    def _push_state(self, h, res, w):
        t = res.transformation
        h.set_state(_cabi.TF_RIGID, self._update_scale, w, t.rot, t.t, t.scale, res.sigma2, res.q)

    def _result_from(self, out):
        rot, t, scale, sigma2, q, _ = out
        return MstepResult(tf.RigidTransformation(rot, t, scale, xp=np), sigma2, q)

    def maximization_step(self, target, estep_res, sigma2_p=None):
        h = self._em_handle(_points(target))
        pt1, p1, px, n_p = estep_res
        return self._result_from(h.mstep(_cabi.TF_RIGID, self._update_scale, pt1, p1, px, n_p))

    @staticmethod
    def _maximization_step(source, target, estep_res, sigma2_p=None, update_scale=True, xp=np):
        """Static form of probreg/cpd.py:160-192 (weighted Procrustes from an EstepResult)."""
        obj = RigidCPD(source, update_scale=update_scale)
        return obj.maximization_step(target, estep_res, sigma2_p)


class AffineCPD(CoherentPointDrift):
    """Affine CPD (x -> B x + t) -- probreg/cpd.py:195-244.

    ``source``: (M, D) array or None; ``tf_init_params``: warm start, keys ``b``/``t``; ``use_cuda``: accepted,
    ignored (module docstring); ``device``/``comm``: see CoherentPointDrift.
    """

    def __init__(self, source=None, tf_init_params=None, use_cuda=False, device=None, comm=None):
        super(AffineCPD, self).__init__(source, use_cuda, device, comm)
        self._tf_type = tf.AffineTransformation
        self._tf_init_params = dict(tf_init_params) if tf_init_params else {}

    def _initialize(self, target):
        dim = self._source.shape[1]
        sigma2 = self._squared_kernel_sum(self._source, target)
        q = 1.0 + target.shape[0] * dim * 0.5 * np.log(sigma2)
        params = dict(self._tf_init_params)
        if len(params) == 0:
            params = {"b": np.identity(dim), "t": np.zeros(dim)}
        params.setdefault("xp", np)
        return MstepResult(self._tf_type(**params), sigma2, q)

    def _push_state(self, h, res, w):
        t = res.transformation
        h.set_state(_cabi.TF_AFFINE, True, w, t.b, t.t, 1.0, res.sigma2, res.q)

    def _result_from(self, out):
        b, t, _, sigma2, q, _ = out
        return MstepResult(tf.AffineTransformation(b, t), sigma2, q)

    def maximization_step(self, target, estep_res, sigma2_p=None):
        h = self._em_handle(_points(target))
        pt1, p1, px, n_p = estep_res
        return self._result_from(h.mstep(_cabi.TF_AFFINE, True, pt1, p1, px, n_p))

    @staticmethod
    def _maximization_step(source, target, estep_res, sigma2_p=None, xp=np):
        """Static form of probreg/cpd.py:219-244."""
        return AffineCPD(source).maximization_step(target, estep_res, sigma2_p)


class NonRigidCPD(CoherentPointDrift):
    """Coherent Point Drift for nonrigid transformation (probreg/cpd.py:247-303).

    ``registration`` keeps G (float32, like ``_math.rbf_kernel``), W and the
    M x M system on the device -- E-step by the CPD kernels, the dense solve of cpd.py:296 by cuSOLVER's LU,
    sigma2 in residual form.  ``maximization_step`` on a caller-supplied EstepResult runs the same solve on the
    device (cpd_nonrigid_mstep) with sigma2 from the reference's three traces.

    ``source``: (M, D) array or None; ``beta``: RBF width of G (denominator 2*beta, as in the reference);
    ``lmd``: weight of the smoothness term; ``use_cuda``: accepted, ignored.

    Extension (no reference counterpart; BASELINE configuration 5): ``low_rank=K`` replaces G by a rank-K
    factorisation Q Bc Q^T found on the device by a seeded randomised range finder (``low_rank_iters`` subspace
    iterations); each M-step is then a K x K solve and nothing of size M x M exists anywhere.  The result carries a
    ``LowRankNonRigidTransformation``.
    """

    def __init__(self, source=None, beta=2.0, lmd=2.0, use_cuda=False, device=None, comm=None, low_rank=None,
                 low_rank_iters=2, low_rank_seed=0):
        super(NonRigidCPD, self).__init__(source, use_cuda, device, comm)
        self._tf_type = tf.NonRigidTransformation
        self._beta = beta
        self._lmd = lmd
        self._low_rank = low_rank
        self._low_rank_iters = low_rank_iters
        self._low_rank_seed = low_rank_seed
        self._tf_obj = None
        self._nr_key = self._nr_src = self._nr_handle = self._nr_factors = None      # what the handle's G / factors were built for
        if not self._source is None:
            self._tf_obj = self._tf_type(None, self._source, self._beta, self.xp, device=self._device)

    def set_source(self, source):
        super(NonRigidCPD, self).set_source(source)
        self._tf_obj = self._tf_type(None, self._source, self._beta, device=self._device)

    def maximization_step(self, target, estep_res, sigma2_p=None):
        """Non-rigid M-step (probreg/cpd.py:284-303) from a caller-supplied EstepResult, on the device
        (cpd_nonrigid_mstep): the M x M (or, with ``low_rank``, K x K) solve, T = Y + G W and sigma2 from the three traces.
        G / its factors are rebuilt only when the source changed since the last call."""
        target = _points(target)
        h = self._nonrigid_handle(target, sigma2_p)
        pt1, p1, px, n_p = estep_res
        sigma2 = h.nonrigid_mstep(pt1, p1, px, sigma2_p)
        self._tf_obj.w = h.nonrigid_w()
        return MstepResult(self._tf_obj, sigma2, sigma2)

    def _nonrigid_handle(self, target, sigma2):
        """Handle with the current source's G (or factors) resident and, for the constrained variant, its priors set."""
        assert self._source is not None, "source is None."
        dim = self._source.shape[1]
        key = (self._beta, self._low_rank, self._low_rank_iters, self._low_rank_seed)
        fresh = (self._em is None or self._em.dim != dim or getattr(self, "_nr_key", None) != key or
                 getattr(self, "_nr_src", None) is None or getattr(self, "_nr_handle", None) is not self._em or
                 not np.array_equal(self._nr_src, self._source))
        self._em_handle(target)                              # uploads source (deterministic internal order) and target
        h = self._em
        if fresh:
            if self._low_rank:
                h.nonrigid_lowrank_begin(self._beta, self._lmd, sigma2, 0.0, self._low_rank, self._low_rank_iters, self._low_rank_seed)
                self._nr_factors = h.nonrigid_lowrank_factors()
                self._tf_obj = tf.LowRankNonRigidTransformation(self._tf_obj.w, self._source, self._beta, self._nr_factors[0],
                                                                self._nr_factors[1], device=self._device)
            else:
                h.nonrigid_begin(self._beta, self._lmd, sigma2, 0.0)
            self._nr_key, self._nr_src, self._nr_handle = key, np.array(self._source, copy=True), h
        else:
            h.nonrigid_restart(self._lmd, sigma2, 0.0)
        prior = self._device_prior()
        if prior is not None:
            self._em.nonrigid_set_prior(*prior)
        return self._em

    def _initialize(self, target):
        dim = self._source.shape[1]
        sigma2 = self._squared_kernel_sum(self._source, target)
        q = 1.0 + target.shape[0] * dim * 0.5 * np.log(sigma2)
        self._tf_obj.w = np.zeros_like(self._source, dtype=np.float64)
        return MstepResult(self._tf_obj, sigma2, q)

    @staticmethod
    def _maximization_step(source, target, estep_res, sigma2_p, tf_obj, lmd, xp=np):
        """Static form of probreg/cpd.py:284-303 (tf_obj supplies beta; its w is updated in place like the reference's)."""
        obj = NonRigidCPD(source, beta=tf_obj._beta, lmd=lmd)
        res = obj.maximization_step(target, estep_res, sigma2_p)
        tf_obj.w = res.transformation.w
        return MstepResult(tf_obj, res.sigma2, res.q)

    def _device_prior(self):
        """(alpha, p1_tilde, px_tilde) for the device loop, or None (ConstrainedNonRigidCPD overrides)."""
        return None

    def _has_device_loop(self):
        # a subclass that brings its own M-step is driven through expectation_step / maximization_step instead
        return type(self).maximization_step in (NonRigidCPD.maximization_step, ConstrainedNonRigidCPD.maximization_step)

    def registration(self, target, w=0.0, maxiter=50, tol=0.001):
        """The loop of probreg/cpd.py:106-120 with G (or its low-rank factors), W, the linear system and its LU
        resident on the GPU (cpd_nonrigid_begin / cpd_nonrigid_lowrank_begin, cpd_nonrigid_step); per iteration only
        sigma2 (== q, cpd.py:303) comes back, plus W when a callback wants the transformation."""
        assert not self._tf_type is None, "transformation type is None."
        target = _points(target)
        res = self._initialize(target)
        if not self._has_device_loop():
            return self._host_loop(target, res, w, maxiter, tol)
        h = self._em
        key = (self._beta, self._low_rank, self._low_rank_iters, self._low_rank_seed)
        if (getattr(self, "_nr_key", None) == key and getattr(self, "_nr_src", None) is not None and self._nr_handle is h
                and np.array_equal(self._nr_src, self._source)):
            h.nonrigid_restart(self._lmd, res.sigma2, w)          # same source as last time: G / the factors are still valid
            if self._low_rank:
                self._tf_obj = tf.LowRankNonRigidTransformation(self._tf_obj.w, self._source, self._beta, self._nr_factors[0],
                                                                self._nr_factors[1], device=self._device)
        else:
            self._nr_key = self._nr_src = None
            if self._low_rank:
                h.nonrigid_lowrank_begin(self._beta, self._lmd, res.sigma2, w, self._low_rank, self._low_rank_iters, self._low_rank_seed)
                self._nr_factors = h.nonrigid_lowrank_factors()
                self._tf_obj = tf.LowRankNonRigidTransformation(self._tf_obj.w, self._source, self._beta, self._nr_factors[0],
                                                                self._nr_factors[1], device=self._device)
            else:
                h.nonrigid_begin(self._beta, self._lmd, res.sigma2, w)
            self._nr_key, self._nr_src, self._nr_handle = key, np.array(self._source, copy=True), h
        prior = self._device_prior()
        if prior is not None:
            h.nonrigid_set_prior(*prior)
        q = res.q
        want_tf = bool(self._callbacks)
        for i in range(maxiter):
            sigma2 = h.nonrigid_step()
            if want_tf:
                self._tf_obj.w = h.nonrigid_w()
            res = MstepResult(self._tf_obj, sigma2, sigma2)
            for c in self._callbacks:
                c(res.transformation)
            log.debug("Iteration: {}, Criteria: {}".format(i, res.q))
            if abs(res.q - q) < tol:
                break
            q = res.q
        if maxiter > 0:
            self._tf_obj.w = h.nonrigid_w()
        return res

    def moved_source(self):
        """The source after the last ``registration``, Y + G W, straight from the device (no M x M product)."""
        assert self._em is not None, "registration has not been run."
        return self._em.nonrigid_moved()

    def _host_loop(self, target, res, w, maxiter, tol):
        q = res.q
        for i in range(maxiter):
            t_source = res.transformation.transform(self._source)
            estep_res = self.expectation_step(t_source, target, res.sigma2, w)
            res = self.maximization_step(target, estep_res, res.sigma2)
            for c in self._callbacks:
                c(res.transformation)
            log.debug("Iteration: {}, Criteria: {}".format(i, res.q))
            if abs(res.q - q) < tol:
                break
            q = res.q
        return res

    def _push_state(self, h, res, w):  # unused: the non-rigid loop is driven from Python
        raise NotImplementedError

    def _result_from(self, out):
        raise NotImplementedError


class ConstrainedNonRigidCPD(NonRigidCPD):
    """Extended CPD with point-correspondence priors (probreg/cpd.py:306-404,
    https://people.mpi-inf.mpg.de/~golyanik/04_DRAFTS/ECPD2016.pdf).

    ``alpha``: trust in the priors (1e-8 = near-hard constraints ... 1 = weak); ``idx_source``/``idx_target``:
    integer arrays of equal length naming the known source/target pairs; the rest as NonRigidCPD.

    The reference materialises a dense M x N indicator matrix for the priors (cpd.py:370-374); its row
    sums and its product with the target are a sparse gather, which is what is computed here.
    """

    def __init__(self, source=None, beta=2.0, lmd=2.0, alpha=1e-8, use_cuda=False, idx_source=None, idx_target=None,
                 device=None, comm=None, low_rank=None, low_rank_iters=2, low_rank_seed=0):
        super(ConstrainedNonRigidCPD, self).__init__(source, beta, lmd, use_cuda, device, comm, low_rank, low_rank_iters,
                                                     low_rank_seed)
        self.alpha = alpha
        self.idx_source, self.idx_target = idx_source, idx_target
        self.p1_tilde = None
        self.px_tilde = None

    def _initialize(self, target):
        res = super(ConstrainedNonRigidCPD, self)._initialize(target)
        self._prior_terms(target)
        return res

    def _prior_terms(self, target):
        """p1_tilde / px_tilde of cpd.py:370-374 as a sparse gather (duplicates count once, like the 0/1 indicator matrix)."""
        m, dim = self._source.shape
        self.p1_tilde = np.zeros(m)
        self.px_tilde = np.zeros((m, dim))
        if self.idx_source is not None and self.idx_target is not None:
            # the reference writes p_tilde[idx_source, idx_target] = 1 (cpd.py:368): NumPy advanced indexing -- the two index arrays
            # broadcast against each other, negative indices count from the end, boolean masks select positions
            n = np.asarray(target).shape[0]

            def as_index(idx, size):
                a = np.asarray(idx)
                if a.dtype == np.bool_:
                    if a.shape != (size,):
                        raise IndexError("boolean index of shape %s does not match the axis of size %d" % (a.shape, size))
                    return np.flatnonzero(a)
                if not np.issubdtype(a.dtype, np.integer):
                    raise IndexError("idx_source / idx_target must be integer or boolean index arrays, got %s" % a.dtype)
                if a.size and (a.min() < -size or a.max() >= size):
                    raise IndexError("index out of bounds for axis of size %d" % size)
                return a.astype(np.intp) % size

            isrc, itgt = np.broadcast_arrays(as_index(self.idx_source, m), as_index(self.idx_target, n))
            pairs = np.unique(np.c_[isrc.ravel(), itgt.ravel()], axis=0)
            np.add.at(self.p1_tilde, pairs[:, 0], 1.0)
            np.add.at(self.px_tilde, pairs[:, 0], np.asarray(target, dtype=np.float64)[pairs[:, 1]])

    def maximization_step(self, target, estep_res, sigma2_p=None):
        """cpd.py:376-404 on the device: NonRigidCPD.maximization_step with the two prior terms (``_device_prior``)."""
        if self.p1_tilde is None:
            self._prior_terms(_points(target))
        return NonRigidCPD.maximization_step(self, target, estep_res, sigma2_p)

    def _device_prior(self):
        return (self.alpha, self.p1_tilde, self.px_tilde)


def registration_cpd(source, target, tf_type_name="rigid", w=0.0, maxiter=50, tol=0.001, callbacks=(),
                     use_cuda=False, **kwargs):
    """One-call CPD registration with the signature of probreg/cpd.py:407-456.

    source, target -- (M, D) / (N, D) arrays (or open3d point clouds), D = 2 or 3
    tf_type_name   -- 'rigid' | 'affine' | 'nonrigid' | 'nonrigid_constrained' (anything else: ValueError)
    w              -- weight of the uniform outlier component, 0 <= w < 1
    maxiter, tol   -- at most maxiter EM iterations; stop once |q - q_prev| < tol
    callbacks      -- callables invoked as cb(transformation) after every iteration
    use_cuda       -- accepted for compatibility, ignored: the H100 kernels are the only implementation
    **kwargs       -- forwarded to the class: update_scale, tf_init_params, beta, lmd, alpha, idx_source,
                      idx_target, and the extensions device= / comm=
    Returns MstepResult(transformation, sigma2, q).
    """
    if tf_type_name == "rigid":
        cpd = RigidCPD(_points(source), use_cuda=use_cuda, **kwargs)
    elif tf_type_name == "affine":
        cpd = AffineCPD(_points(source), use_cuda=use_cuda, **kwargs)
    elif tf_type_name == "nonrigid":
        cpd = NonRigidCPD(_points(source), use_cuda=use_cuda, **kwargs)
    elif tf_type_name == "nonrigid_constrained":
        cpd = ConstrainedNonRigidCPD(_points(source), use_cuda=use_cuda, **kwargs)
    else:
        raise ValueError("Unknown transformation type %s" % tf_type_name)
    cpd.set_callbacks(list(callbacks))
    return cpd.registration(_points(target), w, maxiter, tol)


def registration_cpd_batch(sources, targets, tf_type_name="rigid", w=0.0, maxiter=50, tol=0.001, update_scale=True,
                           tf_init_params=None, device=0):
    """Many independent rigid or affine CPD registrations in one call (no reference counterpart: probreg registers one pair
    per ``registration_cpd`` call).

    sources, targets -- sequences of B arrays (or open3d point clouds); pair k is (sources[k], targets[k]).  Sizes may differ
                        from pair to pair; every pair has the same D, 2 or 3
    tf_type_name     -- 'rigid' | 'affine' ('nonrigid' and anything else: ValueError)
    w, maxiter, tol  -- as in registration_cpd, for every pair
    update_scale     -- RigidCPD's update_scale (rigid only)
    tf_init_params   -- None, or B dicts with the keys registration_cpd takes (rigid: rot / t / scale, affine: b / t); an
                        empty dict or None entry starts that pair from the identity
    device           -- CUDA ordinal

    Each pair gets exactly what ``registration_cpd(source, target, tf_type_name, w, maxiter, tol, update_scale=...,
    tf_init_params=...)`` computes for it without callbacks: sigma2 from the closed form of ``cpd_sigma2_init``, q from
    1 + N D / 2 log sigma2 (probreg/cpd.py:148) and the stop rule |q - q_prev| < tol after an iteration.  Callbacks are not
    offered: the whole batch runs on the device (one CTA per pair, csrc/batch.cuh) with one read-back at the end.  A pair of
    more than 2^16 points in a cloud or 2^26 point pairs (m n) is refused; it belongs to ``registration_cpd``.

    Returns (results, n_iter): a list of B MstepResult (RigidTransformation / AffineTransformation, sigma2, q) and an int array
    of the iterations each pair ran.
    """
    if tf_type_name in ("nonrigid", "nonrigid_constrained"):
        raise ValueError("registration_cpd_batch registers rigid and affine pairs only; use registration_cpd for %s" % tf_type_name)
    if tf_type_name not in ("rigid", "affine"):
        raise ValueError("Unknown transformation type %s" % tf_type_name)
    sources, targets = list(sources), list(targets)
    if len(sources) != len(targets):
        raise ValueError("sources and targets must have the same length, got %d and %d" % (len(sources), len(targets)))
    b = len(sources)
    if b == 0:
        return [], np.zeros(0, dtype=np.int32)
    srcs = [np.asarray(_points(s), dtype=np.float64) for s in sources]
    tgts = [np.asarray(_points(t), dtype=np.float64) for t in targets]
    dim = srcs[0].shape[1] if srcs[0].ndim == 2 else None
    for k in range(b):
        for name, a in (("source", srcs[k]), ("target", tgts[k])):
            if a.ndim != 2 or a.shape[1] != dim:
                raise ValueError("pair %d: the %s has shape %s; every cloud of the batch must be (count, %s)" % (k, name, a.shape, dim))
    if dim not in (2, 3):
        raise ValueError("probreg_b200 supports 2-D and 3-D points, got %s-D" % dim)
    rigid = tf_type_name == "rigid"
    init = None
    if tf_init_params is not None:
        tf_init_params = list(tf_init_params)
        if len(tf_init_params) != b:
            raise ValueError("tf_init_params must hold one dict per pair: %d for %d pairs" % (len(tf_init_params), b))
        init = []
        keys = {"rot", "t", "scale"} if rigid else {"b", "t"}
        for k, params in enumerate(tf_init_params):
            params = dict(params or {})
            params.pop("xp", None)
            bad = set(params) - keys
            if bad:
                raise ValueError("pair %d: unknown tf_init_params key(s) %s for %s CPD" % (k, sorted(bad), tf_type_name))
            lin = params.get("rot" if rigid else "b", np.identity(dim))
            init.append((lin, params.get("t", np.zeros(dim)), params.get("scale", 1.0) if rigid else 1.0))
    src_off = np.r_[0, np.cumsum([s.shape[0] for s in srcs])]
    tgt_off = np.r_[0, np.cumsum([t.shape[0] for t in tgts])]
    out, iters = _cabi.batch_register(np.concatenate(srcs), src_off, np.concatenate(tgts), tgt_off, dim,
                                      _cabi.TF_RIGID if rigid else _cabi.TF_AFFINE, update_scale, w, maxiter, tol, init, device)
    results = []
    for lin, t, scale, sigma2, q, _ in out:
        tf_obj = tf.RigidTransformation(lin, t, scale, xp=np) if rigid else tf.AffineTransformation(lin, t)
        results.append(MstepResult(tf_obj, sigma2, q))
    return results, iters
