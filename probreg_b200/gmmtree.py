"""GMMTree registration (Eckart et al., ECCV 2018) -- the API surface of ``probreg.gmmtree`` with the tree on the H100.

The hierarchical GMM is built on the device from the source (``cpd_gmmtree_build``: per level an EM loop whose E-step evaluates
each point's 8 candidate children, whose log-likelihood runs over the whole level, in FP64 with fixed-order reductions), and the
registration E-step descends the tree on the device for every target point (``cpd_gmmtree_estep``).  The M-step is the
reference's least-squares twist over the nodes, in numpy: it is O(nodes), not O(points).

Departures from the reference, on purpose:
  * the 8^L leaves are seeded from ``np.random.default_rng(seed).integers(0, M, 8**L)`` (``leaf_seeds``), not from Eigen's
    ``std::rand``-based draw, which for L >= 2 reads beyond the indices it drew;
  * pdfs, log-likelihood and moments are FP64 (the reference is float32; at 1M points one float32 ulp of q exceeds lambda_s);
  * each level of the build stops after ``build_maxiter`` EM iterations (the reference loops until converged);
    ``build_iterations`` holds what each level ran;
  * ``MstepResult.q`` is the float residual sum of squares of the least-squares solve (NaN when the system is rank deficient),
    where the reference hands on numpy's array.
"""
from collections import namedtuple

import numpy as np

from . import _cabi
from . import se3_op as so
from . import transformation as tf
from .log import log

EstepResult = namedtuple("EstepResult", ["moments"])
MstepResult = namedtuple("MstepResult", ["transformation", "q"])
MstepResult.__doc__ = """Result of the maximization step: transformation (RigidTransformation from source to target), q (residual)."""

LAMBDA_D = 1.0e-4          # the node-death threshold the reference passes to build_gmmtree (gmmtree.py:51)


def _moment_list(mom):
    """(n_total, 13) moments -> the reference's list of (m0, m1 (3,), m2 (3, 3))"""
    return [(mom[j, 0], mom[j, 1:4], mom[j, 4:13].reshape(3, 3)) for j in range(mom.shape[0])]


class GMMTree(object):
    """GMM Tree

    source -- (M, 3) source cloud (or None, then ``set_source``);  tree_level -- depth L of the tree (1..5);  lambda_c -- pruning
    threshold of the descent (complexity of a node's covariance);  lambda_s -- convergence tolerance of each level of the build;
    tf_init_params -- initial RigidTransformation parameters.  Extensions over the reference: device (CUDA ordinal), seed (of the
    leaf seeds), build_maxiter (EM iterations per level at most).
    """

    def __init__(self, source=None, tree_level=2, lambda_c=0.01, lambda_s=0.001, tf_init_params={}, device=0, seed=0,
                 build_maxiter=1000):
        self._source = None
        self._tree_level = int(tree_level)
        self._lambda_c = lambda_c
        self._lambda_s = lambda_s
        self._tf_type = tf.RigidTransformation
        self._tf_result = self._tf_type(**tf_init_params)
        self._callbacks = []
        self._device = device
        self._seed = seed
        self._build_maxiter = int(build_maxiter)
        self._h = None
        self._nodes = None
        self.build_iterations = None
        self.leaf_seeds = None
        if source is not None:
            self.set_source(source)

    def _handle(self):
        if self._h is None:
            self._h = _cabi.Handle(3, self._device)
        return self._h

    def set_source(self, source):
        """Set the source and build its tree on the device."""
        src = _cabi.as_cloud(source, 3)
        h = self._handle()
        h.set_source(src)
        self._source = src
        self.leaf_seeds = np.random.default_rng(self._seed).integers(0, len(src), 8 ** self._tree_level)
        self.build_iterations = h.gmmtree_build(self._tree_level, self._lambda_s, LAMBDA_D, self.leaf_seeds, self._build_maxiter)
        self._set_nodes(*h.gmmtree_nodes())

    def _set_nodes(self, pi, mu, cov):
        self._nodes = [(pi[j], mu[j], cov[j]) for j in range(len(pi))]
        self._mu = mu
        with np.errstate(invalid="ignore", divide="ignore"):
            self._eig = np.linalg.eigh(cov)            # the M-step's eigh of every node, once per tree

    def set_callbacks(self, callbacks):
        self._callbacks = callbacks

    def expectation_step(self, target):
        """Moments (m0, m1, m2) of `target` per node, each point added to the node its descent ends at."""
        h = self._handle()
        h.set_target(_cabi.as_cloud(target, 3))
        return EstepResult(_moment_list(h.gmmtree_estep(np.identity(3), np.zeros(3), self._lambda_c)))

    def maximization_step(self, estep_res, trans_p):
        """The reference's least-squares twist (gmmtree.py:64-83), vectorised over the nodes; the twist is composed with trans_p."""
        moments = estep_res.moments
        n = len(moments)
        m0 = np.array([m[0] for m in moments], dtype=np.float64)
        m1 = np.array([m[1] for m in moments], dtype=np.float64).reshape(n, 3)
        amat = np.zeros((n, 3, 6))
        bmat = np.zeros((n, 3))
        use = m0 >= np.finfo(np.float32).eps
        if use.any():
            lmd, vec = self._eig[0][use], self._eig[1][use]
            s = m1[use] / m0[use, None]
            with np.errstate(invalid="ignore", divide="ignore"):
                nn = vec * np.sqrt(m0[use, None] / lmd)[:, None, :]          # columns scaled by sqrt(m0 / lambda)
            nt = np.swapaxes(nn, 1, 2)                                         # rows: the scaled eigenvectors
            bmat[use] = np.einsum("nij,nj->ni", nt, self._mu[use]) - np.einsum("nij,nj->ni", nt, s)
            amat[use, :, :3] = np.cross(s[:, None, :], nt)
            amat[use, :, 3:] = nt
        x, res, _, _ = np.linalg.lstsq(amat.reshape(3 * n, 6), bmat.reshape(3 * n), rcond=-1)
        q = float(res[0]) if res.size else float("nan")
        rot, t = so.twist_mul(x, trans_p.rot, trans_p.t)
        return MstepResult(tf.RigidTransformation(rot, t), q)

    def registration(self, target, maxiter=20, tol=1.0e-4):
        """EM on the target (moved by the current transform), gmmtree.py:85-96; returns MstepResult(inverse transform, q).
        The target is uploaded once and each E-step gets the transform; a subclass that overrides ``expectation_step`` is given
        the moved target instead."""
        tgt = _cabi.as_cloud(target, 3)
        direct = type(self).expectation_step is GMMTree.expectation_step
        if direct:
            self._handle().set_target(tgt)
        q, res = None, None
        for i in range(maxiter):
            if direct:
                cur = self._tf_result
                mom = self._h.gmmtree_estep(cur.scale * np.asarray(cur.rot), cur.t, self._lambda_c)
                estep_res = EstepResult(_moment_list(mom))
            else:
                estep_res = self.expectation_step(self._tf_result.transform(tgt))
            res = self.maximization_step(estep_res, self._tf_result)
            self._tf_result = res.transformation
            for c in self._callbacks:
                c(self._tf_result.inverse())
            log.debug("Iteration: {}, Criteria: {}".format(i, res.q))
            if q is not None and abs(res.q - q) < tol:
                break
            q = res.q
        return MstepResult(self._tf_result.inverse(), res.q if res is not None else None)


def registration_gmmtree(source, target, maxiter=20, tol=1.0e-4, callbacks=[], **kwargs):
    """GMMTree registration of source (M, 3) to target (N, 3).

    Keyword args go to GMMTree: tree_level, lambda_c, lambda_s, tf_init_params, device, seed, build_maxiter.
    Returns MstepResult(transformation, q).
    """
    gt = GMMTree(np.asarray(source), **kwargs)
    gt.set_callbacks(callbacks)
    return gt.registration(np.asarray(target), maxiter, tol)
