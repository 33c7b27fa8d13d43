"""Gauss transform on the H100 -- the API of ``probreg.gauss_transform`` (gauss_transform.py:28-60).

    sum_j weights[j] * exp(-||target[i] - source[j]||^2 / h^2)

The reference switches between a direct numpy evaluation (h < sw_h) and the IFGT approximation (eps = 1e-4);
here it is always the exact sum, evaluated by the same tiled pair kernel as the CPD E-step
(cpd_gauss_transform).  ``eps`` and ``sw_h`` are accepted for signature compatibility.
"""
import numpy as np

from . import _cabi


class GaussTransform(object):
    def __init__(self, source, h, eps=1.0e-4, sw_h=0.01, device=0):
        self._source = _cabi.as_cloud(source)
        self._m = self._source.shape[0]
        self._h = float(h)
        self._device = device

    def compute(self, target, weights=None):
        """target: (N, D); weights: (M,) -> (N,), or (K, M) -> (K, N)  (gauss_transform.py:47-60)."""
        tgt = _cabi.as_cloud(target, self._source.shape[1])
        if weights is None:
            weights = np.ones(self._m)
        w = np.ascontiguousarray(weights, dtype=np.float64)
        if w.ndim not in (1, 2):
            raise ValueError("weights.ndim must be 1 or 2.")
        w2 = w.reshape(1, -1) if w.ndim == 1 else w
        if w2.shape[1] != self._m:
            raise ValueError("weights must have one entry per source point")
        out = np.empty((w2.shape[0], tgt.shape[0]))
        _cabi.check(_cabi.lib().cpd_gauss_transform(self._device, _cabi.dptr(self._source), self._m, _cabi.dptr(tgt), tgt.shape[0],
                                                    tgt.shape[1], self._h, _cabi.dptr(w2), w2.shape[0], _cabi.dptr(out)))
        return out[0] if w.ndim == 1 else out
