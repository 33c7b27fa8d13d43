"""probreg_b200 -- the CPD EM hot path of neka-nat/probreg, written for the H100 (sm_90a).

    from probreg_b200 import cpd
    tf_param, sigma2, q = cpd.registration_cpd(source, target)

See the comments of csrc/kernels.cuh for the kernels and INTEGRATION.md for how a probreg checkout binds to them.
"""
from . import bcpd, cost_functions, cpd, features, filterreg, gauss_transform, gaussian_filtering, gmmtree, io, l2dist_regs, log, math_utils, se3_op, transformation  # noqa: F401,E501
from .version import __version__  # noqa: F401
