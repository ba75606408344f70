"""Signal utilities (mirror of /root/reference/src/sionna/phy/signal/utils.py): ``convolve`` on ``sb_convolve``,
normalised DFTs on the OFDM FFT kernels, and the empirical PSD / ACLR on ``sb_ofdm_demodulate`` + ``sb_power_mean``
(``csrc/signal.cu``, DESIGN §3.14)."""
import warnings

import numpy as np
import torch

from ..config import config, dtypes
from ..block import fallback_to_single
from ..._lib import lib, check, ptr, current_stream, SbUnsupportedError

_MAX_FFT = 8192
_warned_show = False


def _dft(x, axis, inverse):
    dev = config.device
    x = torch.as_tensor(x).to(device=dev, dtype=torch.complex64)
    x = x.movedim(axis, -1).contiguous()
    n = x.shape[-1]
    rows = x.numel() // n
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.empty_like(x)
    if inverse:
        check(lib().sb_ofdm_modulate(ptr(x), ptr(out), rows, 1, n, ptr(zero), ptr(zero), n, 0, current_stream()),
              "sb_ofdm_modulate")
    else:
        check(lib().sb_ofdm_demodulate(ptr(x), ptr(out), rows, 1, n, ptr(zero), ptr(zero), n, 0, 0, current_stream()),
              "sb_ofdm_demodulate")
    return out.movedim(-1, axis)


def fft(tensor, axis=-1, precision=None):
    """Normalised DFT ``X_m = 1/sqrt(N) sum_n x_n exp(-j 2 pi m n / N)`` along ``axis`` (signal/utils.py:161-204)."""
    return _dft(tensor, axis, False)


def ifft(tensor, axis=-1, precision=None):
    """Normalised IDFT ``x_n = 1/sqrt(N) sum_m X_m exp(j 2 pi m n / N)`` along ``axis`` (signal/utils.py:206-249)."""
    return _dft(tensor, axis, True)


# ---- convolution ------------------------------------------------------------------------------------------------------
CONV_WINDOW_NORMALIZE, CONV_NORMALIZE, CONV_CONJUGATE = 1, 2, 4     # flags of sb_convolve (include/sionna_b200.h)


def _as_float_tensor(v, name, precision):
    """v on the device, cast to the precision's real or complex dtype; integer or boolean input is a TypeError."""
    if not isinstance(v, torch.Tensor):
        v = torch.as_tensor(np.asarray(v))
    if not (v.dtype.is_floating_point or v.dtype.is_complex):
        raise TypeError(f"{name} must be a real or complex floating-point tensor, not {v.dtype}")
    if v.requires_grad:
        raise NotImplementedError(f"{name}: gradients are not supported (the signal kernels have no backward)")
    kind = "cdtype" if v.dtype.is_complex else "rdtype"
    return v.to(device=config.device, dtype=dtypes[precision]["torch"][kind])


def conv_geometry(padding, n, k):
    """(offset, out_len) of sb_convolve for a padding mode (case-insensitive), input length n and kernel length k."""
    padding = padding.lower()
    assert padding in ("valid", "same", "full"), "Invalid padding method"
    if padding == "full":
        return 0, n + k - 1
    if padding == "same":
        return (k - 1) // 2, n
    if k > n:
        raise ValueError(f"padding='valid' needs a kernel no longer than the input (kernel {k}, input {n})")
    return k - 1, n - k + 1


def filter_rows(x, h, w=None, padding="full", axis=-1, flags=0, precision=None):
    """``sb_convolve`` of x along ``axis`` with the taps prepared on chip from h (window w, ``flags``). x, h and w are
    on the device; x and h must be of the precision's real or complex dtype and w of its real dtype or None (anything
    else is a TypeError, checked here so that no caller hands the kernel elements of another size)."""
    rdt, cdt = dtypes[precision]["torch"]["rdtype"], dtypes[precision]["torch"]["cdtype"]
    for name, v in (("x", x), ("the taps", h)):
        if v.dtype not in (rdt, cdt):
            raise TypeError(f"{name} must be {rdt} or {cdt} for precision '{precision}', not {v.dtype}")
    if w is not None and w.dtype != rdt:
        raise TypeError(f"the window must be {rdt} for precision '{precision}', not {w.dtype}")
    if x.requires_grad:
        raise NotImplementedError("convolve: gradients are not supported (the signal kernels have no backward)")
    if h.dim() != 1:
        raise ValueError(f"the kernel must be one-dimensional, got shape {tuple(h.shape)}")
    x = x.movedim(axis, -1).contiguous()
    n, k = x.shape[-1], h.shape[0]
    offset, out_len = conv_geometry(padding, n, k)
    rows = x.numel() // n if n else 0
    out_dtype = dtypes[precision]["torch"]["cdtype" if (x.is_complex() or h.is_complex()) else "rdtype"]
    y = torch.empty(tuple(x.shape[:-1]) + (out_len,), dtype=out_dtype, device=x.device)
    h = h.contiguous()
    w = None if w is None else w.contiguous()
    check(lib().sb_convolve(ptr(x), int(x.is_complex()), ptr(h), int(h.is_complex()), ptr(w), ptr(y),
                            int(precision == "double"), rows, n, k, offset, out_len, flags, current_stream()),
          "sb_convolve")
    return y.movedim(-1, axis)


def convolve(inp, ker, padding="full", axis=-1, precision=None):
    """Filters ``inp`` [..., N] by convolving it with ``ker`` [K] along ``axis`` (signal/utils.py:11-159).

    Both inputs are cast to the precision's real or complex dtype; the output is complex if either input is. Padding
    (case-insensitive): "full" (N + K - 1 outputs), "same" (N outputs, centred on tap (K - 1) // 2, which is what the
    reference's TF "SAME" with a padded kernel gives; for K <= N this is ``np.convolve(..., "same")``, and for K > N it
    still returns N outputs) or "valid" (N - K + 1 outputs). Unlike the reference, "valid" with K > N raises
    ``ValueError`` and integer inputs raise ``TypeError``. Double precision runs natively in float64. No autograd:
    inputs with ``requires_grad`` raise ``NotImplementedError``."""
    precision = precision or config.precision
    x = _as_float_tensor(inp, "inp", precision)
    h = _as_float_tensor(ker, "ker", precision)
    return filter_rows(x, h, padding=padding, axis=axis, precision=precision)


# ---- PSD and ACLR -----------------------------------------------------------------------------------------------------
def _linspace_f32(start, stop, num):
    """tf.linspace in float32: start + i (stop - start) / (num - 1), the last point exactly stop."""
    start, stop = np.float32(start), np.float32(stop)
    if num == 1:
        return np.array([start], np.float32)
    step = (stop - start) / np.float32(num - 1)
    out = start + np.arange(num, dtype=np.float32) * step
    out[-1] = stop
    return out


_tables = {}


def _device_table(key, make):
    """A small constant host table, copied to the device once per key (the device is part of the key). Callers
    must not modify it."""
    if key not in _tables:
        _tables[key] = torch.from_numpy(make()).to(key[-1])
    return _tables[key]


def _power_mean(x):
    """(1 / rows) sum_r |x[r, j]|^2 of a complex64 [rows, N] device tensor through sb_power_mean (deterministic)."""
    rows, n = x.shape
    psd = torch.empty(n, dtype=torch.float32, device=x.device)
    ws_bytes = lib().sb_power_mean_workspace_bytes(rows, n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
    check(lib().sb_power_mean(ptr(x), ptr(psd), rows, n, ptr(ws), ws_bytes, current_stream()), "sb_power_mean")
    return psd


def empirical_psd(x, show=True, oversampling=1.0, ylim=(-30, 3), precision=None):
    """Empirical power spectral density of ``x`` [..., N] along the last dimension, averaged over all other dimensions
    (signal/utils.py:251-311): ``psd = mean |fftshift(fft(x))|^2`` with the normalised DFT, and ``freqs`` the float32
    ``linspace(-oversampling / 2, oversampling / 2, N)``. Returns ``(freqs, psd)``, both [N].

    Plotting is not provided: ``show=True`` (the reference's default) returns the values and warns once that no plot
    is drawn. 1 <= N <= 8192 (the FFT kernel's range). ``precision="double"`` computes in single precision and widens
    the outputs (``PrecisionWarning``)."""
    global _warned_show
    if show and not _warned_show:
        _warned_show = True
        warnings.warn("empirical_psd: no plot is drawn (plotting is not provided); the values are returned",
                      stacklevel=2)
    double = fallback_to_single("empirical_psd", precision)
    dev = config.device
    x = torch.as_tensor(x).to(device=dev, dtype=torch.complex64)
    n = x.shape[-1]
    if not 1 <= n <= _MAX_FFT:
        raise SbUnsupportedError(f"empirical_psd: N = {n}, supported are 1 <= N <= {_MAX_FFT} (the FFT's range)")
    x = x.reshape(-1, n).contiguous()
    rows = x.shape[0]
    if rows == 0:
        raise ValueError("empirical_psd: x holds no rows to average over")
    spec = torch.empty_like(x)
    zero = _device_table(("zero", dev), lambda: np.zeros(1, np.int32))
    check(lib().sb_ofdm_demodulate(ptr(x), ptr(spec), rows, 1, n, ptr(zero), ptr(zero), n, 0, 1, current_stream()),
          "sb_ofdm_demodulate")
    psd = _power_mean(spec)
    freqs = _device_table(("freqs", n, float(oversampling), dev),
                          lambda: _linspace_f32(-0.5 * oversampling, 0.5 * oversampling, n)).clone()
    if double:
        return freqs.to(torch.float64), psd.to(torch.float64)
    return freqs, psd


def empirical_aclr(x, oversampling=1.0, f_min=-0.5, f_max=0.5, precision=None):
    """Empirical adjacent channel leakage ratio of ``x`` [..., N] (signal/utils.py:313-368): the PSD summed over the
    frequencies strictly below ``f_min`` or strictly above ``f_max``, over its sum strictly inside (f_min, f_max).
    Summed on the host in float64; returns a Python ``float`` (linear scale)."""
    freqs, psd = empirical_psd(x, show=False, oversampling=oversampling, precision=precision)
    f = freqs.cpu().numpy()
    p = psd.cpu().numpy().astype(np.float64)
    lo, hi = np.asarray(f_min, f.dtype), np.asarray(f_max, f.dtype)
    p_out = p[(f < lo) | (f > hi)].sum()
    p_in = p[(f > lo) & (f < hi)].sum()
    return float(p_out / p_in)
