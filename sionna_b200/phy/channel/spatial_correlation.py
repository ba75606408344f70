"""Spatial correlation of flat-fading channels (mirror of the reference's channel/spatial_correlation.py:12-195).

``KroneckerModel`` and ``PerColumnModel`` run on ``sb_flat_fading``; their Cholesky factors come from ``sb_chol_lower``
(fp32) and are kept per assigned tensor until it changes (identity, version counter, device and dtype), so a fixed
correlation is factored once. A correlation matrix that is not positive definite in fp32 gives NaN in its own factor
and in the channels it correlates, without a host synchronisation. Matrices of any other type than a torch tensor
(NumPy arrays, lists) are factored on every call, since in-place edits to them cannot be seen."""
from abc import abstractmethod

import numpy as np
import torch

from ..block import Object, fallback_to_single
from ..config import config
from ..._lib import lib, check, ptr, current_stream


def cholesky(r):
    """Lower Cholesky factors of ``r [..., n, n]`` (complex, n <= 128) on the device, complex64, by ``sb_chol_lower``."""
    r = torch.as_tensor(r).to(device=config.device, dtype=torch.complex64).contiguous()
    n = r.shape[-1]
    l = torch.empty_like(r)
    check(lib().sb_chol_lower(ptr(r), ptr(l), r.numel() // max(n * n, 1), n, current_stream()), "sb_chol_lower")
    return l


class _Factor:
    """The Cholesky factor of one assigned correlation tensor (None stays None)."""

    def __init__(self, r):
        self.r = r
        self._key, self._l = None, None

    def get(self):
        r = self.r
        if r is None:
            return None
        if not isinstance(r, torch.Tensor):
            return cholesky(np.asarray(r))
        key = (r._version, r.device, r.dtype, config.device)
        if key != self._key:
            self._l, self._key = cholesky(r), key
        return self._l


def _prod(shape):
    return int(np.prod(shape)) if len(shape) else 1


def factor_set(l, set_lead, out_lead, tail):
    """(contiguous factors, stride) for sb_flat_fading: factors ``l [*set_lead, *tail]`` broadcast against the channel
    uses ``out_lead``. One set for every use gives stride 0, one per use in order stride 1; any other pattern is
    expanded to ``out_lead`` (the factor of an expanded R is the expanded factor)."""
    n = _prod(set_lead)
    if n == 1:
        return l.reshape(tail).contiguous(), 0
    if n == _prod(out_lead):
        return l.reshape((n,) + tuple(tail)).contiguous(), 1
    return l.expand(tuple(out_lead) + tuple(tail)).contiguous(), 1


class SpatialCorrelation(Object):
    """Abstract spatial correlation of a flat-fading channel: ``__call__(h)`` maps spatially uncorrelated channel
    coefficients to correlated ones (spatial_correlation.py:12-40)."""

    @abstractmethod
    def __call__(self, h, *args, **kwargs):
        return NotImplemented


class _FactorModel(SpatialCorrelation):
    """The models ``sb_flat_fading`` computes: ``plan(h_lead, M, K)`` gives the channel uses' leading shape and the
    kernel's factor arguments."""

    def __call__(self, h):
        from .flat_fading_channel import flat_fading
        h = torch.as_tensor(h)
        wide = h.dtype == torch.complex128
        if wide:
            fallback_to_single(type(self).__name__, "double")
        h = h.to(device=config.device, dtype=torch.complex64)
        m, k = h.shape[-2], h.shape[-1]
        lead, fac = self.plan(tuple(h.shape[:-2]), m, k)
        out = flat_fading(lead, m, k, h=h, want_h=True, **fac)[1]
        return out.to(torch.complex128) if wide else out


class KroneckerModel(_FactorModel):
    r"""Kronecker model ``H_corr = L_rx H L_tx^H`` with ``L = cholesky(R)`` (spatial_correlation.py:42-122).
    ``r_tx [..., K, K]`` and ``r_rx [..., M, M]`` (either may be None) broadcast against ``h [..., M, K]``'s leading
    dimensions. Limits: K <= 128 with ``r_tx``, M <= 128 with ``r_rx`` and M K <= 16384."""

    def __init__(self, r_tx=None, r_rx=None, precision=None):
        super().__init__(precision=precision)
        self.r_tx = r_tx
        self.r_rx = r_rx

    @property
    def r_tx(self):
        """[..., K, K] complex: get/set the transmit correlation matrices."""
        return self._tx.r

    @r_tx.setter
    def r_tx(self, value):
        self._tx = _Factor(value)

    @property
    def r_rx(self):
        """[..., M, M] complex: get/set the receive correlation matrices."""
        return self._rx.r

    @r_rx.setter
    def r_rx(self, value):
        self._rx = _Factor(value)

    def plan(self, h_lead, m, k):
        l_tx, l_rx = self._tx.get(), self._rx.get()
        shapes = [h_lead] + [tuple(l.shape[:-2]) for l in (l_tx, l_rx) if l is not None]
        lead = tuple(torch.broadcast_shapes(*shapes))
        fac = {}
        if l_tx is not None:
            fac["tx"] = factor_set(l_tx, l_tx.shape[:-2], lead, (k, k))
        if l_rx is not None:
            fac["rx"] = factor_set(l_rx, l_rx.shape[:-2], lead, (m, m))
        return lead, fac


class PerColumnModel(_FactorModel):
    r"""Per-column model ``h_k <- L_k h_k`` for every column k of ``h [..., M, K]`` with ``L_k = cholesky(R_k)``
    (spatial_correlation.py:124-195). ``r_rx [..., M, M]`` broadcasts against ``h``'s leading dimensions followed by K:
    ``[M, M]`` for every column, ``[K, M, M]`` one per column, ``[..., K, M, M]`` one per column and channel use.
    Limits: M <= 128 and M K <= 16384."""

    def __init__(self, r_rx, precision=None):
        super().__init__(precision=precision)
        self.r_rx = r_rx

    @property
    def r_rx(self):
        """[..., M, M] complex: get/set the receive correlation matrices."""
        return self._rx.r

    @r_rx.setter
    def r_rx(self, value):
        self._rx = _Factor(value)

    def plan(self, h_lead, m, k):
        l_rx = self._rx.get()
        if l_rx is None:
            return h_lead, {}
        set_lead = tuple(l_rx.shape[:-2])
        full = tuple(torch.broadcast_shapes(tuple(h_lead) + (k,), set_lead))
        lead = full[:-1]
        if full[-1] != k:
            raise ValueError(f"r_rx with leading shape {set_lead} does not broadcast against {k} columns of h")
        if _prod(set_lead) in (1, k) and set_lead[-1:] in ((), (1,), (k,)) and _prod(set_lead[:-1]) == 1:
            l = l_rx.reshape(-1, m, m).expand(k, m, m).contiguous()          # one [K, M, M] set for every use
            return lead, {"rx": (l, 0), "per_column": True}
        l, stride = factor_set(l_rx, set_lead, full, (m, m))
        return lead, {"rx": (l.reshape(-1, k, m, m), stride), "per_column": True}
