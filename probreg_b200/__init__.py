"""probreg_b200 -- the CPD EM hot path of neka-nat/probreg, written for the H100 (sm_90a).

    from probreg_b200 import cpd
    tf_param, sigma2, q = cpd.registration_cpd(source, target)

See the comments of csrc/kernels.cuh for the kernels and INTEGRATION.md for how a probreg checkout binds to them.
"""
from . import bcpd, cpd, gauss_transform, io, log, math_utils, transformation  # noqa: F401
from .version import __version__  # noqa: F401
