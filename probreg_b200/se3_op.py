"""Twist helpers of ``probreg.se3_op`` used by GMMTree's M-step (reference: se3_op.py), without the transforms3d dependency."""
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
