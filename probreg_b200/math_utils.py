"""The two ``probreg.math_utils`` helpers the CPD path uses, on the GPU.

* ``squared_kernel_sum``  probreg/math_utils.py:28-29 -> ``_math.squared_kernel`` (cc/math_utils.cc:15)
* ``rbf_kernel``          probreg/math_utils.py:36-37 -> ``_math.rbf_kernel``     (cc/math_utils.cc:17-19)

The reference materialises an nx x ny float32 matrix for the first one just to sum it; here it
is the O(nx + ny) closed form evaluated in FP64 on the device (cpd_squared_kernel_sum).
"""
import ctypes

import numpy as np

from . import _cabi


def squared_kernel_sum(x, y, device=0):
    xa, ya = _cabi.as_cloud(x), _cabi.as_cloud(y)
    if xa.shape[1] != ya.shape[1]:
        raise ValueError("x and y must have same dimensions.")
    out = ctypes.c_double()
    _cabi.check(_cabi.lib().cpd_squared_kernel_sum(device, _cabi.dptr(xa), xa.shape[0], _cabi.dptr(ya), ya.shape[0],
                                                   xa.shape[1], ctypes.byref(out)))
    return out.value


def rbf_kernel(x, y, beta, device=0):
    xa, ya = _cabi.as_cloud(x), _cabi.as_cloud(y)
    if xa.shape[1] != ya.shape[1]:
        raise ValueError("x and y must have same dimensions.")
    out = np.empty((xa.shape[0], ya.shape[0]), dtype=np.float32)
    _cabi.check(_cabi.lib().cpd_rbf_kernel(device, _cabi.dptr(xa), xa.shape[0], _cabi.dptr(ya), ya.shape[0], xa.shape[1],
                                           float(beta), out.ctypes.data_as(ctypes.POINTER(ctypes.c_float))))
    return out


def inverse_multiquadric_kernel(x, y, c=1.0, device=0):
    """probreg/math_utils.py:50-51 -> ``_math.inverse_multiquadric_kernel`` (cc/math_utils.cc:37-39), float32, on the device."""
    xa, ya = _cabi.as_cloud(x), _cabi.as_cloud(y)
    if xa.shape[1] != ya.shape[1]:
        raise ValueError("x and y must have same dimensions.")
    out = np.empty((xa.shape[0], ya.shape[0]), dtype=np.float32)
    _cabi.check(_cabi.lib().cpd_imq_kernel(device, _cabi.dptr(xa), xa.shape[0], _cabi.dptr(ya), ya.shape[0], xa.shape[1],
                                           float(c), out.ctypes.data_as(ctypes.POINTER(ctypes.c_float))))
    return out


def compute_rmse(source, target_tree):
    """probreg/math_utils.py:32-33: mean nearest-neighbour distance of ``source`` in a scipy cKDTree of the target."""
    return float(np.sum(target_tree.query(source)[0]) / source.shape[0])
