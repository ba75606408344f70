"""NumPy restatement of sionna.phy.signal (signal/utils.py, filter.py, window.py): convolution in the generic
(offset, out_len) form of sb_convolve, the pulse and window formulas, Filter.call's tap preparation, the empirical PSD
and ACLR. Everything is evaluated in float64 / complex128 unless ``dtype`` asks for float32 / complex64 (the "f32
evaluation" the fp32 envelope of oracle.parity compares the kernels against)."""
import numpy as np


def geometry(padding, n, k):
    """(offset, out_len) of padding "full", "same" or "valid" for input length n and kernel length k."""
    return {"full": (0, n + k - 1), "same": ((k - 1) // 2, n), "valid": (k - 1, n - k + 1)}[padding.lower()]


def convolve(x, h, padding="full", single=False):
    """y[..., m] = sum_k h[k] x[..., m + offset - k] (x = 0 outside [0, N)), m < out_len, along the last axis, summed
    over k in ascending order in complex128 / float64, or in complex64 / float32 with single=True."""
    cplx = np.iscomplexobj(x) or np.iscomplexobj(h)
    dt = (np.complex64 if cplx else np.float32) if single else (np.complex128 if cplx else np.float64)
    x = np.asarray(x).astype(dt if np.iscomplexobj(x) else np.dtype(dt).type(0).real.dtype)
    h = np.asarray(h).astype(dt if np.iscomplexobj(h) else np.dtype(dt).type(0).real.dtype)
    n, k = x.shape[-1], h.shape[0]
    offset, out_len = geometry(padding, n, k)
    full = np.zeros(x.shape[:-1] + (n + k - 1,), dt)
    for i in range(k):
        full[..., i:i + n] += h[i] * x
    return full[..., offset:offset + out_len]


# ---- pulses and windows (float64) -------------------------------------------------------------------------------------
def sampling_times(span, sps):
    """Sample times in symbol durations of a filter of span * sps taps, forced odd, centred on 0."""
    length = 2 * (span * sps // 2) + 1
    return np.arange(-(length // 2), length - length // 2) / sps


def raised_cosine(t, beta):
    t = np.abs(np.asarray(t, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        h = np.sinc(t) * np.cos(np.pi * beta * t) / (1 - (2 * beta * t) ** 2)
    if beta > 0:
        h[np.isclose(t, 1 / (2 * beta), rtol=0, atol=1e-12)] = np.pi / 4 * np.sinc(1 / (2 * beta))
    return h


def root_raised_cosine(t, beta):
    t = np.abs(np.asarray(t, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        h = (np.sin(np.pi * t * (1 - beta)) + 4 * beta * t * np.cos(np.pi * t * (1 + beta))) / (
            np.pi * t * (1 - (4 * beta * t) ** 2))
    if beta > 0:
        h[np.isclose(t, 1 / (4 * beta), rtol=0, atol=1e-12)] = beta / np.sqrt(2) * (
            (1 + 2 / np.pi) * np.sin(np.pi / (4 * beta)) + (1 - 2 / np.pi) * np.cos(np.pi / (4 * beta)))
    h[t == 0] = 1 + beta * (4 / np.pi - 1)
    return h


def sinc(t):
    return np.sinc(np.asarray(t, np.float64))


def window(kind, n):
    """Periodic Hann / Hamming / Blackman window of length n (w_n over n / N, 0 <= n < N)."""
    x = np.arange(n) / n
    if kind == "hann":
        return np.sin(np.pi * x) ** 2
    if kind == "hamming":
        return 25 / 46 - 21 / 46 * np.cos(2 * np.pi * x)
    return (7938 - 9240 * np.cos(2 * np.pi * x) + 1430 * np.cos(4 * np.pi * x)) / 18608


def prepare_taps(h, w=None, window_normalize=False, normalize=True, conjugate=False, single=False):
    """Filter.call's taps: h w~ (w~ = w / sqrt(mean(w^2)) if window_normalize), / sqrt(sum |.|^2) if normalize, then
    conjugated if asked (filter.py:268-285, window.py:145-163)."""
    cplx = np.iscomplexobj(h)
    rt = np.float32 if single else np.float64
    h = np.asarray(h).astype((np.complex64 if single else np.complex128) if cplx else rt)
    if w is not None:
        w = np.asarray(w).astype(rt)
        if window_normalize:
            w = w / np.sqrt(np.mean(w * w))
        h = h * w
    if normalize:
        h = h / np.sqrt(np.sum(np.abs(h) ** 2))
    if conjugate and cplx:
        h = np.conj(h)
    return h


# ---- PSD and ACLR -----------------------------------------------------------------------------------------------------
def linspace_f32(start, stop, num):
    """tf.linspace in float32: start + i * ((stop - start) / (num - 1)), the last point exactly stop."""
    start, stop = np.float32(start), np.float32(stop)
    if num == 1:
        return np.array([start], np.float32)
    out = start + np.arange(num, dtype=np.float32) * ((stop - start) / np.float32(num - 1))
    out[-1] = stop
    return out


def psd(x, oversampling=1.0, single=False):
    """(freqs, psd): mean over all leading axes of |fftshift(fft(x) / sqrt(N))|^2 (signal/utils.py:251-311)."""
    x = np.asarray(x).astype(np.complex64 if single else np.complex128)
    n = x.shape[-1]
    spec = np.fft.fftshift(np.fft.fft(x.reshape(-1, n), axis=-1), axes=-1) / np.sqrt(n)
    if single:
        spec = spec.astype(np.complex64)
    p = np.mean(np.abs(spec) ** 2, axis=0)
    return linspace_f32(-0.5 * oversampling, 0.5 * oversampling, n), p


def aclr(freqs, p, f_min=-0.5, f_max=0.5):
    """Out-of-band (f < f_min or f > f_max) over in-band (f_min < f < f_max) power."""
    f = np.asarray(freqs)
    lo, hi = np.asarray(f_min, f.dtype), np.asarray(f_max, f.dtype)
    p = np.asarray(p, np.float64)
    return float(p[(f < lo) | (f > hi)].sum() / p[(f > lo) & (f < hi)].sum())
