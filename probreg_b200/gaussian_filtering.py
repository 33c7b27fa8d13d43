"""``probreg.gaussian_filtering`` on the H100: the permutohedral lattice of the reference (third_party/permutohedral), built and
applied on the device (``cpd_lattice_filter``) and bit-identical to the reference's x86-64 build: the same lattice size and the
same float32 filtered values."""
import numpy as np

from . import _cabi


class Permutohedral(object):
    """Permutohedral(p, with_blur): the lattice over the points p (n x d, d = 2 or 3; rounded to float32 as the reference's
    binding rounds them).  filter(v, start) filters v (n x vs, vs = 1..8) and returns n x vs float32; like the reference it
    splats every row whatever `start` is."""

    def __init__(self, p, with_blur=True, device=0):
        self._p = np.ascontiguousarray(p, dtype=np.float32)
        if self._p.ndim != 2 or self._p.shape[1] not in (2, 3):
            raise ValueError("the lattice features must be (n x 2) or (n x 3), got shape %s" % (self._p.shape,))
        self._with_blur = bool(with_blur)
        self._device = device
        self._size = _cabi.lattice_filter(self._p, None, self._with_blur, device)[1]

    def get_lattice_size(self):
        return self._size

    def filter(self, v, start=0):
        return _cabi.lattice_filter(self._p, v, self._with_blur, self._device)[0]
