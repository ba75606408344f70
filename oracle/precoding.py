"""Oracle: transmit precoding. TEST INFRASTRUCTURE (NumPy). Literal restatements of the reference's
src/sionna/phy:
  mimo/precoding.py:12-89 (rzf_precoding_matrix), 91-155 (cbf_precoding_matrix), 157-245 (rzf_precoder)
  ofdm/precoding.py:139-156 / 246-295 (desired-channel gather), 297-346 (effective channel), 348-369 (tx power),
  118-177 (RZFPrecoder), 417-446 / 486-510 / 547-566 (RZF / CBF / Eye precoded channels)       -> ofdm_precode
``dtype=np.complex128`` is the oracle; ``np.complex64`` evaluates the same sequence in single precision, the reference's
own fp32 error envelope (the convention of oracle/mimo.py).
"""
import numpy as np

from .ofdm import _cholesky_solve, _herm


def _rdt(cdt):
    return np.float64 if np.dtype(cdt) == np.complex128 else np.float32


def _normalize(g):
    """divide_no_nan(g, ||column||): a zero column stays zero."""
    norm = np.sqrt(np.sum(np.abs(g) ** 2, axis=-2, keepdims=True)).astype(g.dtype)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(norm == 0, np.zeros((), g.dtype), g / np.where(norm == 0, 1, norm))


def rzf_precoding_matrix(h, alpha=0., dtype=np.complex128):
    """h [..., K, M], alpha [...] aligned with h's leading dimensions from the left -> g [..., M, K]."""
    h = np.asarray(h).astype(dtype)
    g = h @ _herm(h)                                                     # [..., K, K]
    alpha = np.asarray(alpha).astype(_rdt(dtype))
    alpha = alpha.reshape(alpha.shape + (1,) * (g.ndim - alpha.ndim))    # expand_to_rank(alpha, rank(g), axis=-1)
    g = g + (alpha * np.eye(g.shape[-1])).astype(dtype)
    return _normalize(_herm(_cholesky_solve(g, h)))


def cbf_precoding_matrix(h, dtype=np.complex128):
    return _normalize(_herm(np.asarray(h).astype(dtype)))


def rzf_precoder(x, h, alpha=0., dtype=np.complex128):
    """(G x [..., M], G [..., M, K])."""
    g = rzf_precoding_matrix(h, alpha, dtype)
    return (g @ np.asarray(x).astype(dtype)[..., None])[..., 0], g


def desired_channels(h_hat, precoding_ind):
    """[B, RX, RA, TX, M, S, F] -> [B, TX, S, F, num_rx_per_tx * RA, M]: transpose, gather(precoding_ind, axis=1,
    batch_dims=1), flatten, transpose (ofdm/precoding.py:268-284)."""
    h = np.transpose(h_hat, [3, 1, 2, 4, 5, 6, 0])                       # [TX, RX, RA, M, S, F, B]
    h = np.stack([h[j][precoding_ind[j]] for j in range(h.shape[0])])  # [TX, RPT, RA, M, S, F, B]
    h = h.reshape((h.shape[0], -1) + h.shape[3:])                        # [TX, RPT * RA, M, S, F, B]
    return np.transpose(h, [5, 0, 3, 4, 1, 2])


def ofdm_precode(kind, h, precoding_ind, eff_ind, x=None, h_hat=None, alpha=0., alpha_left=False, tx_power=None,
                 dtype=np.complex128):
    """(x_precoded [B, TX, M, S, F] or None, h_eff [B, RX, RA, TX, K, S, NE]) for kind "rzf" / "cbf" / "eye".
    alpha broadcasts to [B, TX, S, F] aligned on the right (RZFPrecoder) or, alpha_left, on the left
    (RZFPrecodedChannel); tx_power is [B, TX, K, S, F] or its first n dimensions (None: no power scale)."""
    h = np.asarray(h).astype(dtype)
    b, rx, ra, tx, m, s_, f_ = h.shape
    if kind == "eye":
        g = np.broadcast_to(np.eye(m, dtype=dtype), (b, tx, s_, f_, m, m))
    else:
        hd = desired_channels(h if h_hat is None else np.asarray(h_hat).astype(dtype), precoding_ind)
        if kind == "rzf":
            al = np.asarray(alpha).astype(_rdt(dtype))
            if alpha_left:
                al = al.reshape(al.shape + (1,) * (4 - al.ndim))
            g = rzf_precoding_matrix(hd, np.broadcast_to(al, (b, tx, s_, f_)), dtype)
        else:
            g = cbf_precoding_matrix(hd, dtype)                          # [B, TX, S, F, M, K]
    xp = None
    if x is not None:
        xt = np.transpose(np.asarray(x).astype(dtype), [0, 1, 3, 4, 2])[..., None]     # [B, TX, S, F, K, 1]
        xp = np.transpose((g @ xt)[..., 0], [0, 1, 4, 2, 3])
    if tx_power is not None:                                             # apply_tx_power
        p = np.asarray(tx_power).astype(_rdt(dtype))
        p = p.reshape(p.shape + (1,) * (6 - p.ndim))
        p = np.broadcast_to(np.transpose(p, [0, 1, 3, 4, 5, 2]), g.shape)
        g = np.sqrt(p).astype(dtype) * g
    ht = np.transpose(h, [0, 1, 3, 5, 6, 2, 4])                          # [B, RX, TX, S, F, RA, M]
    h_eff = np.transpose(ht @ g[:, None], [0, 1, 5, 2, 6, 3, 4])         # [B, RX, RA, TX, K, S, F]
    return xp, h_eff[..., np.asarray(eff_ind)]
