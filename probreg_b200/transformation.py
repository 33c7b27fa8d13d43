"""Transformation value types returned by the CPD classes.

Same class names, constructor arguments, attributes (``rot``/``t``/``scale``, ``b``/``t``,
``w``/``g``, ``xp``) and methods (``transform``, ``inverse``, ``__mul__``) as
probreg/transformation.py:18-102, so callbacks and user code written against the reference
keep working.  They are plain host-side (numpy) value objects: inside the EM loop the
transform is applied on the device by ``pack_kernel`` (csrc/kernels.cuh), not through these.
"""
import abc

import numpy as np

try:  # open3d is optional here (the reference imports it unconditionally, transformation.py:5)
    import open3d as _o3

    _Vector3dVector = _o3.utility.Vector3dVector
except Exception:  # pragma: no cover - open3d is absent in the build image
    class _Vector3dVector(object):
        """Placeholder so that ``isinstance(points, array_type)`` is simply False."""

from . import math_utils as mu


class Transformation(abc.ABC):
    def __init__(self, xp=np):
        self.xp = xp

    def transform(self, points, array_type=_Vector3dVector):
        # transformation.py:23-26: open3d vectors round-trip, arrays pass straight through
        if isinstance(points, array_type):
            return array_type(self._transform(np.asarray(points)))
        return self._transform(points)

    @abc.abstractmethod
    def _transform(self, points):
        return points


class RigidTransformation(Transformation):
    """x -> scale * rot @ x + t   (transformation.py:33-60)."""

    def __init__(self, rot=None, t=None, scale=1.0, xp=np):
        super(RigidTransformation, self).__init__(xp)
        self.rot = np.identity(3) if rot is None else rot
        self.t = np.zeros(3) if t is None else t
        self.scale = scale

    def _transform(self, points):
        return self.scale * np.dot(points, np.asarray(self.rot).T) + self.t

    def inverse(self):
        rt = np.asarray(self.rot).T
        return RigidTransformation(rt, -np.dot(rt, self.t) / self.scale, 1.0 / self.scale)

    def __mul__(self, other):
        return RigidTransformation(np.dot(self.rot, other.rot), self.t + self.scale * np.dot(self.rot, other.t),
                                   self.scale * other.scale)


class AffineTransformation(Transformation):
    """x -> b @ x + t   (transformation.py:63-78)."""

    def __init__(self, b=None, t=None, xp=np):
        super(AffineTransformation, self).__init__(xp)
        self.b = np.identity(3) if b is None else b
        self.t = np.zeros(3) if t is None else t

    def _transform(self, points):
        return np.dot(points, np.asarray(self.b).T) + self.t


class NonRigidTransformation(Transformation):
    """x_i -> x_i + (G w)_i with G the RBF Gram matrix of the source (transformation.py:81-102).

    ``g`` is built by the CUDA RBF kernel (math_utils.rbf_kernel -> cpd_rbf_kernel), float32 like
    the reference's ``_math.rbf_kernel`` -- on first use rather than in the constructor (the reference builds it
    eagerly, transformation.py:96): the device-resident EM loop keeps its own G and a caller that only wants
    ``w`` or the final moved points never pays for an M x M host array.
    """

    def __init__(self, w, points, beta=2.0, xp=np, device=0):
        super(NonRigidTransformation, self).__init__(xp)
        self._points = points
        self._beta = beta
        self._g = None
        self._device = device            # CUDA ordinal of the registration that owns this map (extension over the reference)
        self.w = w

    @property
    def g(self):
        if self._g is None:              # built lazily, on the owner's GPU (not always GPU 0: multi-rank runs)
            self._g = mu.rbf_kernel(self._points, self._points, self._beta, device=self._device)
        return self._g

    @g.setter
    def g(self, value):
        self._g = value

    def _transform(self, points):
        return points + np.dot(self.g, self.w)


class LowRankNonRigidTransformation(NonRigidTransformation):
    """The same map with G ~= q bcore q^T (rank K): x_i -> x_i + (q (bcore (q^T w)))_i.

    Produced by ``NonRigidCPD(..., low_rank=K)``; no reference counterpart (the reference only has the dense G).
    ``q`` (M x K, orthonormal columns) and ``bcore`` (K x K) come from the device (cpd_nonrigid_lowrank_get).
    ``g`` stays available (dense, built on first use) for code written against the reference's attribute.
    """

    def __init__(self, w, points, beta, q, bcore, xp=np, device=0):
        super(LowRankNonRigidTransformation, self).__init__(w, points, beta, xp, device)
        self.q = q
        self.bcore = bcore

    def _transform(self, points):
        return points + np.dot(self.q, np.dot(self.bcore, np.dot(self.q.T, self.w)))


class CombinedTransformation(Transformation):
    """x -> rigid(x + v): a per-point displacement followed by a similarity (transformation.py:105-121; BCPD)."""

    def __init__(self, rot=None, t=None, scale=1.0, v=0.0):
        super(CombinedTransformation, self).__init__()
        self.rigid_trans = RigidTransformation(np.identity(3) if rot is None else rot, np.zeros(3) if t is None else t, scale)
        self.v = v

    def _transform(self, points):
        return self.rigid_trans._transform(points + self.v)


class TPSTransformation(Transformation):
    """Thin-plate spline x -> [1, x, U(x) P] [a; v] (transformation.py:124-160): a ((D + 1) x D) the affine part, v
    ((n - D - 1) x D) the warp on the null space P of [1, control_pts], U the TPS kernel (math_utils.tps_kernel, float32 on the
    device) against the n control points."""

    def __init__(self, a, v, control_pts, kernel=mu.tps_kernel):
        super(TPSTransformation, self).__init__()
        self.a = a
        self.v = v
        self.control_pts = control_pts
        self._kernel = kernel

    def prepare(self, landmarks):
        """(basis (m x (n + 1)), kernel ((n - D - 1) x (n - D - 1))) of `landmarks`: they depend on the landmarks and the control
        points only, not on a or v."""
        control_pts = self.control_pts
        m, d = landmarks.shape
        n, _ = control_pts.shape
        pm = np.c_[np.ones((m, 1)), landmarks]
        pn = np.c_[np.ones((n, 1)), control_pts]
        u, _, _ = np.linalg.svd(pn)
        pp = u[:, d + 1:]
        kk = self._kernel(control_pts, control_pts)
        uu = self._kernel(landmarks, control_pts)
        basis = np.c_[pm, np.dot(uu, pp)]
        kernel = np.dot(pp.T, np.dot(kk, pp))
        return basis, kernel

    def transform_basis(self, basis):
        return np.dot(basis, np.r_[self.a, self.v])

    def _transform(self, points):
        basis, _ = self.prepare(points)
        return self.transform_basis(basis)
