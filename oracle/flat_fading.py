"""Oracle: flat-fading MIMO channels restated in NumPy from the formulas (TEST INFRASTRUCTURE).

Every function takes `dtype`: complex128 is the float64 reference, complex64 the single-precision evaluation whose error
against it sets the envelope of `oracle.parity.envelope`.
  exp_corr      R[i, j] = a^(i - j) (i >= j), conj(a)^(j - i) (i < j)                     (exponential model)
  one_ring      R[l, m] = exp(j 2 pi d (l - m) sin phi) exp(-s^2 / 2 (2 pi d (l - m) cos phi)^2)   (one-ring model)
  chol          lower L with L L^H = R (complex64: written out, numpy.linalg would compute it in double)
  kronecker     L_rx (H L_tx^H)   (tx factor first, either may be None)
  per_column    column k of H times L[k]
  apply         y = H x
  draw          the kernel's unit complex normal stream of [num, M, K] from (seed, offset): oracle.rng.awgn / sqrt 2
"""
import numpy as np

from . import rng as R


def exp_corr(a, n, dtype=np.complex128):
    """[..., n, n] exponential correlation matrices, one per element of a."""
    a = np.asarray(a, dtype=np.complex128)[..., None, None]
    i = np.arange(n)[:, None]
    j = np.arange(n)[None, :]
    with np.errstate(invalid="ignore"):
        low = a ** np.maximum(i - j, 0)
        up = np.conj(a) ** np.maximum(j - i, 0)
    r = np.where(i >= j, low, up)
    r = np.where(i == j, 1.0 + 0j, r)                     # a = 0: 0^0 = 1
    return r.astype(dtype)


def one_ring(phi_deg, num_ant, d_h=0.5, sigma_phi_deg=15.0, dtype=np.complex128):
    """[..., num_ant, num_ant] one-ring covariance matrices of a uniform linear array, one per angle."""
    phi = np.deg2rad(np.asarray(phi_deg, dtype=np.float64))[..., None, None]
    s = np.deg2rad(float(sigma_phi_deg))
    lm = (np.arange(num_ant)[:, None] - np.arange(num_ant)[None, :]).astype(np.float64)
    u = 2 * np.pi * d_h * lm
    r = np.exp(1j * u * np.sin(phi)) * np.exp(-0.5 * (s * u * np.cos(phi)) ** 2)
    return r.astype(dtype)


def chol(r, dtype=np.complex128):
    """Lower L with L L^H = R. numpy.linalg computes single-precision inputs in double precision (and numpy's complex64
    products may fuse multiply-adds), so the complex64 evaluation is written out in float32 operations, each rounded:
    the column-by-column (Cholesky-Crout) order, d_j = r_jj - sum_k |l_jk|^2, l_ij = (r_ij - sum_k l_ik conj(l_jk)) / l_jj."""
    r = np.asarray(r).astype(dtype)
    if dtype == np.complex128:
        return np.linalg.cholesky(r)
    n = r.shape[-1]
    lr = np.zeros(r.shape, np.float32)
    li = np.zeros(r.shape, np.float32)
    with np.errstate(invalid="ignore"):
        for j in range(n):
            d = r[..., j, j].real.astype(np.float32)
            vr = r[..., j + 1:, j].real.astype(np.float32)
            vi = r[..., j + 1:, j].imag.astype(np.float32)
            for k in range(j):
                ar, ai = lr[..., j, k], li[..., j, k]
                d = d - (ar * ar + ai * ai)
                br, bi = lr[..., j + 1:, k], li[..., j + 1:, k]
                vr = vr - (br * ar[..., None] + bi * ai[..., None])
                vi = vi - (bi * ar[..., None] - br * ai[..., None])
            d = np.sqrt(d)
            lr[..., j, j] = d
            lr[..., j + 1:, j] = vr / d[..., None]
            li[..., j + 1:, j] = vi / d[..., None]
    return (lr + 1j * li).astype(np.complex64)


def kronecker(h, l_tx=None, l_rx=None, dtype=np.complex128):
    h = np.asarray(h).astype(dtype)
    if l_tx is not None:
        h = h @ np.conj(np.swapaxes(np.asarray(l_tx).astype(dtype), -1, -2))
    if l_rx is not None:
        h = np.asarray(l_rx).astype(dtype) @ h
    return h


def per_column(h, l, dtype=np.complex128):
    """h [..., M, K], l [..., K, M, M] (broadcast) -> column k of h times l[..., k, :, :]."""
    h = np.asarray(h).astype(dtype)
    hc = np.swapaxes(h, -1, -2)[..., None]                # [..., K, M, 1]
    return np.swapaxes((np.asarray(l).astype(dtype) @ hc)[..., 0], -1, -2)


def apply(h, x, dtype=np.complex128):
    return (np.asarray(h).astype(dtype) @ np.asarray(x).astype(dtype)[..., None])[..., 0]


def draw(seed, offset, num, m, k):
    """The kernel's draw of h [num, m, k] (complex128, before its float32 rounding)."""
    return (R.awgn(seed, offset, num * m * k) * np.sqrt(0.5)).reshape(num, m, k)
