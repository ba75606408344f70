"""MIMO equalisation (mirror of /root/reference/src/sionna/phy/mimo/equalization.py:11-466): LMMSE, ZF and MF."""
import torch

from ..config import config
from ..._lib import lib, check, ptr, current_stream


def lmmse_equalizer(y, h, s, whiten_interference=True, precision=None):
    r"""LMMSE equaliser for ``y = H x + n`` with ``E[n n^H] = S``: returns the unbiased soft symbols
    ``x_hat = diag(G H)^-1 G y`` with ``G = H^H (H H^H + S)^-1`` and the effective noise variances
    ``no_eff = diag(diag(GH)^-1 - I)`` (equalization.py:101-233). The interference is whitened first with the Cholesky
    factor of S, then ``G = (H_w^H H_w + I)^-1 H_w^H`` is obtained by a second Cholesky factorisation
    (``whiten_interference=True``, the reference default); ``whiten_interference=False`` applies
    ``G = H^H (H H^H + S)^-1`` directly (:83-90).

    y [..., M], h [..., M, K], s [..., M, M] -> x_hat [..., K] complex, no_eff [..., K] real."""
    from ..block import fallback_to_single
    if fallback_to_single("lmmse_equalizer", precision):
        x_hat, no_eff = lmmse_equalizer(y, h, s, whiten_interference, "single")
        return x_hat.to(torch.complex128), no_eff.to(torch.float64)
    dev = config.device
    y = torch.as_tensor(y).to(device=dev, dtype=torch.complex64)
    h = torch.as_tensor(h).to(device=dev, dtype=torch.complex64)
    s = torch.as_tensor(s).to(device=dev, dtype=torch.complex64)
    m, k = h.shape[-2], h.shape[-1]
    lead = torch.broadcast_shapes(y.shape[:-1], h.shape[:-2], s.shape[:-2])
    y = y.expand(*lead, m).contiguous()
    h = h.expand(*lead, m, k).contiguous()
    s = s.expand(*lead, m, m).contiguous()
    num = y.numel() // m
    x_hat = torch.empty(*lead, k, dtype=torch.complex64, device=dev)
    no_eff = torch.empty(*lead, k, dtype=torch.float32, device=dev)
    if whiten_interference:
        check(lib().sb_lmmse_equalize(ptr(y), ptr(h), ptr(s), ptr(x_hat), ptr(no_eff), num, m, k, current_stream()),
              "sb_lmmse_equalize")
    else:                                                      # G = H^H (H H^H + S)^-1 without whitening (:83-90, :199-200)
        check(lib().sb_mimo_linalg(3, ptr(y), ptr(h), ptr(s), ptr(x_hat), ptr(no_eff), num, m, k, current_stream()),
              "sb_mimo_linalg")
    return x_hat, no_eff


def _c64(x, dev):
    return torch.as_tensor(x).to(device=dev, dtype=torch.complex64)


def lmmse_matrix(h, s=None, precision=None):
    r"""LMMSE equalisation matrix ``G = H^H (H H^H + S)^-1`` (``s=None``: ``S = I``, computed as
    ``(H^H H + I)^-1 H^H``), mimo/equalization.py:11-99. h [..., M, K], s [..., M, M] -> g [..., K, M]."""
    from ..block import fallback_to_single
    if fallback_to_single("lmmse_matrix", precision):
        return lmmse_matrix(h, s, "single").to(torch.complex128)
    dev = config.device
    h = _c64(h, dev)
    m, k = h.shape[-2], h.shape[-1]
    lead = h.shape[:-2] if s is None else torch.broadcast_shapes(h.shape[:-2], torch.as_tensor(s).shape[:-2])
    h = h.expand(*lead, m, k).contiguous()
    sd = None if s is None else _c64(s, dev).expand(*lead, m, m).contiguous()
    g = torch.empty(*lead, k, m, dtype=torch.complex64, device=dev)
    check(lib().sb_mimo_linalg(2, None, ptr(h), ptr(sd), ptr(g), None, h.numel() // (m * k), m, k, current_stream()),
          "sb_mimo_linalg")
    return g



def _dense_equalizer(name, mode, y, h, s, precision):
    """x_hat [..., K], no_eff [..., K] of sb_mimo_linalg mode 4 (ZF) or 5 (MF) with the broadcasting of
    ``lmmse_equalizer``."""
    from ..block import fallback_to_single
    if fallback_to_single(name, precision):
        x_hat, no_eff = _dense_equalizer(name, mode, y, h, s, "single")
        return x_hat.to(torch.complex128), no_eff.to(torch.float64)
    dev = config.device
    y, h, s = _c64(y, dev), _c64(h, dev), _c64(s, dev)
    m, k = h.shape[-2], h.shape[-1]
    lead = torch.broadcast_shapes(y.shape[:-1], h.shape[:-2], s.shape[:-2])
    y = y.expand(*lead, m).contiguous()
    h = h.expand(*lead, m, k).contiguous()
    s = s.expand(*lead, m, m).contiguous()
    x_hat = torch.empty(*lead, k, dtype=torch.complex64, device=dev)
    no_eff = torch.empty(*lead, k, dtype=torch.float32, device=dev)
    check(lib().sb_mimo_linalg(mode, ptr(y), ptr(h), ptr(s), ptr(x_hat), ptr(no_eff), y.numel() // m, m, k,
                               current_stream()), "sb_mimo_linalg")
    return x_hat, no_eff


def zf_equalizer(y, h, s, precision=None):
    r"""ZF equaliser for ``y = H x + n`` with ``E[n n^H] = S`` (equalization.py:235-343): ``x_hat = G y`` with
    ``G = matrix_pinv(H) = (H^H H)^-1 H^H`` and ``no_eff = Re diag(G S G^H)``; ``sb_mimo_linalg`` mode 4.

    y [..., M], h [..., M, K], s [..., M, M] -> x_hat [..., K] complex, no_eff [..., K] real."""
    return _dense_equalizer("zf_equalizer", 4, y, h, s, precision)


def mf_equalizer(y, h, s, precision=None):
    r"""Matched-filter equaliser (equalization.py:345-466): ``x_hat = G y`` with ``G = diag(H^H H)^-1 H^H`` and
    ``no_eff = |diag((I - G H)(I - G H)^H + G S G^H)|``; ``sb_mimo_linalg`` mode 5.

    y [..., M], h [..., M, K], s [..., M, M] -> x_hat [..., K] complex, no_eff [..., K] real."""
    return _dense_equalizer("mf_equalizer", 5, y, h, s, precision)
