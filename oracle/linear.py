"""Oracle: ZF and MF equalisation, the pseudo-inverse and the symbol demapper. TEST INFRASTRUCTURE (NumPy). Literal
restatements of /root/reference/src/sionna/phy:
  utils/linalg.py (matrix_pinv)                          -> matrix_pinv
  mimo/equalization.py:235-343 (zf_equalizer)            -> zf_equalizer
  mimo/equalization.py:345-466 (mf_equalizer)            -> mf_equalizer
  mapping.py:776-792 (SymbolDemapper.call)               -> symbol_demap
  ofdm/equalization.py:109-462 (OFDMEqualizer + ZF / MF / LMMSE without whitening)  -> ofdm_equalize
Every function evaluates the reference's step sequence in the precision of its inputs (or of `dtype`): complex128 /
float64 is the oracle, complex64 / float32 the reference's own single-precision error envelope, as
oracle.ofdm.lmmse_equalizer_cholesky does for the LMMSE tests.
"""
import numpy as np

from .ofdm import _cholesky_solve, _herm, _ofdm_lmmse, lmmse_equalizer_cholesky


def matrix_pinv(h):
    """cholesky_solve(chol(H^H H), H^H): [..., M, K] -> [..., K, M]."""
    return _cholesky_solve(_herm(h) @ h, _herm(h))


def zf_equalizer(y, h, s):
    """G = matrix_pinv(H), x_hat = G y, no_eff = Re diag(G S G^H)."""
    g = matrix_pinv(h)
    x_hat = (g @ y[..., None])[..., 0]
    return x_hat, np.real(np.diagonal(g @ s @ _herm(g), axis1=-2, axis2=-1))


def mf_equalizer(y, h, s):
    """B = H^H H, G = diag(B)^-1 H^H, x_hat = G y, no_eff = |diag((I - G H)(I - G H)^H + G S G^H)|."""
    hth = _herm(h) @ h
    one = np.ones((), h.dtype)
    d = one / np.diagonal(hth, axis1=-2, axis2=-1)
    g = d[..., :, None] * _herm(h)
    x_hat = (g @ y[..., None])[..., 0]
    gsg = g @ s @ _herm(g)
    i_gh = np.eye(h.shape[-1], dtype=h.dtype) - g @ h
    return x_hat, np.abs(np.diagonal(i_gh @ _herm(i_gh) + gsg, axis1=-2, axis2=-1))


def symbol_demap(y, no, points, prior=None, hard_out=False, dtype=np.float64):
    """e = -|y - c|^2 / no (+ prior) over the points, then log_softmax(e) (e - max - log sum exp(e - max)) [..., n, P]
    or the first argmax [..., n]. no is expanded with trailing dimensions to y's rank (expand_to_rank(.., -1)), prior
    with leading ones."""
    cdt = np.complex128 if np.dtype(dtype) == np.float64 else np.complex64
    y = np.asarray(y).astype(cdt)
    d = np.abs(y[..., None] - np.asarray(points).astype(cdt))
    no = np.asarray(no, dtype)
    no = no.reshape(no.shape + (1,) * (d.ndim - no.ndim))
    e = -(d ** 2) / no
    if prior is not None:
        e = e + np.asarray(prior, dtype)
    if hard_out:
        return np.argmax(e, axis=-1)
    m = np.max(e, axis=-1, keepdims=True)
    return (e - m) - np.log(np.sum(np.exp(e - m), axis=-1, keepdims=True))


OFDM_EQUALIZERS = {
    "lmmse-no-whitening": lambda y, h, s: lmmse_equalizer_cholesky(y, h, s, whiten_interference=False),
    "zf": zf_equalizer,
    "mf": mf_equalizer,
}


def ofdm_equalize(y_eff, h_hat, err_var, no, mask, sm, equalizer, dtype=np.complex128):
    """OFDMEqualizer.call with the equaliser `equalizer` (a name of OFDM_EQUALIZERS) through the LMMSE oracle's
    pre- and post-processing (S assembly, stream re-ordering, data-symbol gather) in precision `dtype`.
    -> x_hat, no_eff [B, tx, st, num_data]."""
    rdt = np.float64 if np.dtype(dtype) == np.complex128 else np.float32
    return _ofdm_lmmse(y_eff, h_hat, err_var, no, mask, sm, dtype, rdt, OFDM_EQUALIZERS[equalizer])
