"""Twist and quaternion helpers of ``probreg.se3_op`` (reference: se3_op.py), used by GMMTree's M-step and GMMReg's rigid cost,
without the transforms3d dependency."""
import numpy as np


def skew(x):
    """3 x 3 skew-symmetric matrix of the cross product with x."""
    return np.array([[0.0, -x[2], x[1]], [x[2], 0.0, -x[0]], [-x[1], x[0], 0.0]])


def twist_trans(tw, linear=False):
    """(rotation, translation) of the twist tw = (omega (3), v (3)); linear: first-order rotation I + [omega]x."""
    if linear:
        return np.identity(3) + skew(tw[:3]), tw[3:]
    twd = np.linalg.norm(tw[:3])
    if twd == 0.0:
        return np.identity(3), tw[3:]
    ntw = tw[:3] / twd
    c, s = np.cos(twd), np.sin(twd)
    tr = c * np.identity(3) + (1.0 - c) * np.outer(ntw, ntw) + s * skew(ntw)
    return tr, tw[3:]


def twist_mul(tw, rot, t, linear=False):
    """The twist applied after (rot, t): (tr rot, tr t + tt)."""
    tr, tt = twist_trans(tw, linear=linear)
    return np.dot(tr, rot), np.dot(t, tr.T) + tt


_FLOAT_EPS = np.finfo(np.float64).eps


def quat2mat(q):
    """Rotation matrix of the quaternion q = (w, x, y, z), which need not be normalised (transforms3d.quaternions.quat2mat's
    formula: R = I + (2 / |q|^2) A(q)); the identity when |q|^2 is below machine epsilon."""
    w, x, y, z = q
    nq = w * w + x * x + y * y + z * z
    if nq < _FLOAT_EPS:
        return np.identity(3)
    s = 2.0 / nq
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return np.array([[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]])


def diff_rot_from_quaternion(q):
    """dR(q)/dq as a (4, 3, 3) array, d_rot[k] = dR/dq_k, with R = quat2mat(q) -- the values of probreg's se3_op.py:62-…

    With R = I + (2 / N) A(q), N = |q|^2: the off-diagonal entries are (2 / N) dA/dq_k - 2 q_k R / N^2 (the exact derivative has
    R / N: the two agree for unit q), and the diagonal entries are the exact derivative, except that dR_22/dq_2 and dR_22/dq_3
    carry the reference's factors (x^2 + y^2) and (w^2 + z^2) where the exact ones are (w^2 + z^2) and (x^2 + y^2); the two agree
    when q_2 = q_3 = 0 or x^2 + y^2 = w^2 + z^2.  Kept as the reference has it: the rigid GMMReg optimiser follows this gradient.
    """
    q = np.asarray(q, dtype=np.float64)
    w, x, y, z = q
    rot = quat2mat(q)
    q2 = np.square(q)
    n = q2.sum()
    n2 = n * n
    da = np.array([
        [[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]],              # dA/dw
        [[0.0, y, z], [y, -2.0 * x, -w], [z, w, -2.0 * x]],      # dA/dx
        [[-2.0 * y, x, w], [x, 0.0, z], [-w, z, -2.0 * y]],      # dA/dy
        [[-2.0 * z, -w, x], [w, -2.0 * z, y], [x, y, 0.0]],      # dA/dz
    ])
    d_rot = 2.0 / n * da
    off = ~np.eye(3, dtype=bool)
    d_rot[:, off] -= 2.0 * q[:, None] * rot[off][None, :] / n2
    diag_a = np.array([-(q2[2] + q2[3]), -(q2[1] + q2[3]), -(q2[1] + q2[2])])    # A_ii
    for i in range(3):
        d_rot[:, i, i] = 2.0 / n * da[:, i, i] - 4.0 * q * diag_a[i] / n2
    d_rot[2, 2, 2] = -4.0 * y * (q2[1] + q2[2]) / n2
    d_rot[3, 2, 2] = 4.0 * z * (q2[3] + q2[0]) / n2
    return d_rot
