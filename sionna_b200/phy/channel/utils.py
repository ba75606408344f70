"""Correlation-matrix helpers of the channel models (mirror of the reference's channel/utils.py:1489-1651). They are
set-up-time tables, not a hot path: built in float64 NumPy on the host, then cast to the precision and placed on
``config.device``."""
import warnings

import numpy as np
import torch

from ..config import config, dtypes


def _to_device(r, precision):
    cdtype = dtypes[precision or config.precision]["torch"]["cdtype"]
    return torch.from_numpy(np.ascontiguousarray(r)).to(device=config.device, dtype=cdtype)


def _hermitian_toeplitz(col):
    """[..., n, n] with R[i, j] = col[i - j] for i >= j and conj(col[j - i]) above the diagonal."""
    n = col.shape[-1]
    d = np.arange(n)[:, None] - np.arange(n)[None, :]
    return np.where(d >= 0, col[..., np.abs(d)], np.conj(col[..., np.abs(d)]))


def exp_corr_mat(a, n, precision=None):
    r"""Exponential correlation matrices ``R[i, j] = a^(i - j)`` for ``i >= j`` and ``conj(a)^(j - i)`` above the
    diagonal, one per element of ``a`` (any shape, complex, ``|a| < 1``): ``[..., n, n]``. ``a = 0`` gives the identity.
    Raises ``ValueError`` if any ``|a| >= 1`` (the reference's ``InvalidArgumentError``)."""
    a = np.asarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, dtype=np.complex128)
    if np.any(np.abs(a) >= 1):
        raise ValueError("The absolute value of the elements of `a` must be smaller than one")
    col = np.ones(a.shape + (int(n),), np.complex128)
    for i in range(1, int(n)):
        col[..., i] = col[..., i - 1] * a
    return _to_device(_hermitian_toeplitz(col), precision)


def one_ring_corr_mat(phi_deg, num_ant, d_h=0.5, sigma_phi_deg=15, precision=None):
    r"""One-ring covariance matrices of a uniform linear array (Eq. 2.24 of Bjornson, Hoydis, Sanguinetti, "Massive
    MIMO Networks", 2017): ``R[l, m] = exp(j 2 pi d_h (l - m) sin(phi)) exp(-sigma^2 / 2 (2 pi d_h (l - m) cos(phi))^2)``
    for the arrival angle ``phi`` (degrees, any shape), antenna spacing ``d_h`` (wavelengths) and angular standard
    deviation ``sigma_phi_deg`` (degrees): ``[..., num_ant, num_ant]``. Warns for ``sigma_phi_deg > 15``, where the
    approximation does not hold. Near endfire (``phi`` close to +-90 degrees) the matrices are close to rank one, and
    singular even in float64."""
    if sigma_phi_deg > 15:
        warnings.warn("sigma_phi_deg should be smaller than 15.")
    phi = np.deg2rad(np.asarray(phi_deg.detach().cpu().numpy() if isinstance(phi_deg, torch.Tensor) else phi_deg,
                                dtype=np.float64))[..., None]
    sigma = np.deg2rad(float(sigma_phi_deg))
    d = 2 * np.pi * float(d_h) * np.arange(int(num_ant), dtype=np.float64)
    col = np.exp(1j * d * np.sin(phi)) * np.exp(-0.5 * (sigma * d * np.cos(phi)) ** 2)
    return _to_device(_hermitian_toeplitz(col), precision)
