"""Pulse-shaping filters (mirror of /root/reference/src/sionna/phy/signal/filter.py) on ``sb_convolve``
(``csrc/signal.cu``): the raw coefficients, the window and the flags go to the kernel, which prepares the taps on chip
(window, unit-energy normalisation, conjugation, in ``Filter.call``'s order, filter.py:268-285) on every call. So a
reassigned or in-place modified ``coefficients`` tensor takes effect on the next call; nothing is cached."""
import numpy as np
import torch

from ..block import Block
from .utils import filter_rows, empirical_aclr, CONV_WINDOW_NORMALIZE, CONV_NORMALIZE, CONV_CONJUGATE
from .window import Window, HannWindow, HammingWindow, BlackmanWindow

_WINDOWS = {"hann": HannWindow, "hamming": HammingWindow, "blackman": BlackmanWindow}


class Filter(Block):
    """Abstract filter of ``length`` K = ``span_in_symbols`` * ``samples_per_symbol`` (plus one if even), applied to
    ``x`` [..., N] by discrete convolution along the last dimension (filter.py:13-285).

    Parameters: ``span_in_symbols``, ``samples_per_symbol``, ``window`` (None, a :class:`Window`, "hann", "hamming" or
    "blackman"), ``normalize`` (unit energy, default True), ``precision``. Input: ``x``, ``padding`` ("full", "same" or
    "valid", see :func:`convolve`), ``conjugate`` (apply the conjugate taps). Output: [..., M], complex if ``x`` or the
    coefficients are. Double precision runs natively in float64.

    Deviations: ``show`` raises ``NotImplementedError`` (no plotting); a window given by name is created with the
    filter's precision (the reference uses the global one and then asserts that they match); ``aclr`` pads the taps to
    max(1024, K) points (the reference fails for K > 1024) and computes the PSD in single precision, from complex64
    taps as the reference does, so it warns in no precision; there is no autograd: coefficients or inputs with
    ``requires_grad`` raise ``NotImplementedError``."""
    _native_double = True

    def __init__(self, span_in_symbols, samples_per_symbol, window=None, normalize=True, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert span_in_symbols > 0, "span_in_symbols must be positive"
        self._span_in_symbols = span_in_symbols
        assert samples_per_symbol > 0, "samples_per_symbol must be positive"
        self._samples_per_symbol = samples_per_symbol
        self.window = window
        assert isinstance(normalize, bool), "normalize must be bool"
        self._normalize = normalize
        self._coefficients = None

    @property
    def span_in_symbols(self):
        """int: Filter span in symbols."""
        return self._span_in_symbols

    @property
    def samples_per_symbol(self):
        """int: Number of samples per symbol, i.e., the oversampling factor."""
        return self._samples_per_symbol

    @property
    def length(self):
        """int: Filter length in samples (span_in_symbols * samples_per_symbol, forced odd)."""
        n = self._span_in_symbols * self._samples_per_symbol
        return 2 * (n // 2) + 1

    @property
    def window(self):
        """:class:`Window`: Get/set the window applied to the filter coefficients."""
        return self._window

    @window.setter
    def window(self, value):
        if isinstance(value, str):
            if value not in _WINDOWS:
                raise AssertionError("Invalid window type")
            value = _WINDOWS[value](precision=self.precision)
        elif not (isinstance(value, Window) or value is None):
            raise AssertionError("Invalid window type")
        if value is not None:
            assert value.precision == self._precision, "Window and Filter must have the same precision."
            if not value.built:                          # build the coefficients for this length (filter.py:141-142)
                value.build((self.length,))
                value._built = True
            self._window_taps(value)
        self._window = value

    def _window_taps(self, window):
        """The window's raw coefficients, checked against the filter length; None without a window."""
        if window is None:
            return None
        w = window.coefficients
        if w.is_complex():
            raise TypeError("window coefficients must be real")
        if w.shape[0] != self.length:
            raise ValueError(f"the window has {w.shape[0]} coefficients, the filter {self.length}")
        return w

    @property
    def normalize(self):
        """bool: If True, the filter is normalized to have unit power."""
        return self._normalize

    @property
    def coefficients(self):
        """[K], float or complex: Set/get the raw filter coefficients."""
        return self._coefficients

    @coefficients.setter
    def coefficients(self, v):
        self._coefficients = self._cast_or_check_precision(v)

    @property
    def sampling_times(self):
        """[K], numpy.float32: Sampling times in multiples of the symbol duration."""
        n_min = -(self.length // 2)
        t = np.arange(n_min, n_min + self.length, dtype=np.float32)
        t /= self.samples_per_symbol
        return t

    def show(self, response="impulse", scale="lin"):
        """Not provided: this package has no plotting (filter.py:173-236)."""
        raise NotImplementedError("Filter.show: plotting is not provided")

    def _flags(self):
        f = CONV_NORMALIZE if self._normalize else 0
        if self._window is not None and self._window.normalize:
            f |= CONV_WINDOW_NORMALIZE
        return f

    def _filter(self, x, padding, flags):
        h = self._coefficients
        w = self._window_taps(self._window)
        if h.requires_grad or (w is not None and w.requires_grad):
            raise NotImplementedError("Filter: gradients are not supported (the signal kernels have no backward)")
        return filter_rows(x, h, w, padding=padding, flags=flags, precision=self.precision)

    @property
    def aclr(self):
        """float: ACLR (linear) of the filter used for pulse shaping of i.i.d. symbols, in-band [-0.5, 0.5]
        (filter.py:238-266): the prepared taps (from ``sb_convolve`` on a unit impulse) zero-padded to 1024 points."""
        impulse = torch.ones(1, dtype=self.rdtype, device=self.device)
        h = self._filter(impulse, "full", self._flags())
        c = torch.zeros(max(1024, h.shape[0]), dtype=torch.complex64, device=self.device)
        c[:h.shape[0]] = h.to(torch.complex64)
        return empirical_aclr(c, oversampling=self._samples_per_symbol, precision="single")

    def call(self, x, padding="full", conjugate=False):
        flags = self._flags() | (CONV_CONJUGATE if conjugate else 0)
        return self._filter(x, padding, flags)


class RaisedCosineFilter(Filter):
    """Raised-cosine filter (filter.py:287-405) with roll-off ``beta`` in [0, 1]:
    h(t) = pi / (4T) sinc(1 / (2 beta)) at t = +-T / (2 beta), else 1/T sinc(t/T) cos(pi beta t / T) /
    (1 - (2 beta t / T)^2). Coefficients in float32 NumPy, as in the reference. Unlike the reference, ``precision``
    is honoured (the reference drops it through a keyword typo, filter.py:378)."""

    def __init__(self, span_in_symbols, samples_per_symbol, beta, window=None, normalize=True, precision=None,
                 **kwargs):
        super().__init__(span_in_symbols, samples_per_symbol, window=window, normalize=normalize, precision=precision,
                         **kwargs)
        assert 0 <= beta <= 1, "beta must be from the intervall [0,1]"
        self._beta = beta
        self.coefficients = raised_cosine(self.sampling_times, 1.0, self.beta)

    @property
    def beta(self):
        """float: Roll-off factor."""
        return self._beta


class RootRaisedCosineFilter(Filter):
    """Root-raised-cosine filter (filter.py:408-531) with roll-off ``beta`` in [0, 1]:
    h(0) = 1/T (1 + beta (4/pi - 1)); h(+-T/(4 beta)) = beta / (T sqrt 2) [(1 + 2/pi) sin(pi / (4 beta)) + (1 - 2/pi)
    cos(pi / (4 beta))]; else 1/T [sin(pi t/T (1 - beta)) + 4 beta t/T cos(pi t/T (1 + beta))] /
    [pi t/T (1 - (4 beta t / T)^2)]. Coefficients in float32 NumPy, as in the reference."""

    def __init__(self, span_in_symbols, samples_per_symbol, beta, window=None, normalize=True, precision=None,
                 **kwargs):
        super().__init__(span_in_symbols, samples_per_symbol, window=window, normalize=normalize, precision=precision,
                         **kwargs)
        assert 0 <= beta <= 1, "beta must be from the intervall [0,1]"
        self._beta = beta
        self.coefficients = root_raised_cosine(self.sampling_times, 1.0, self.beta)

    @property
    def beta(self):
        """float: Roll-off factor."""
        return self._beta


class SincFilter(Filter):
    """Sinc filter h(t) = 1/T sinc(t/T) (filter.py:534-624)."""

    def __init__(self, span_in_symbols, samples_per_symbol, window=None, normalize=True, precision=None, **kwargs):
        super().__init__(span_in_symbols, samples_per_symbol, window=window, normalize=normalize, precision=precision,
                         **kwargs)
        self.coefficients = 1 / 1.0 * np.sinc(self.sampling_times / 1.0)


class CustomFilter(Filter):
    """Filter with user-given ``coefficients`` [K], real or complex, K odd and equal to the length implied by
    ``samples_per_symbol`` (filter.py:627-707)."""

    def __init__(self, samples_per_symbol, coefficients, window=None, normalize=True, precision=None, **kwargs):
        assert samples_per_symbol > 0, "samples_per_symbol must be positive"
        n = coefficients.shape[-1]
        assert n % 2 == 1, "The number of coefficients must be odd"
        super().__init__(n // samples_per_symbol, samples_per_symbol, window=window, normalize=normalize,
                         precision=precision, **kwargs)
        self.coefficients = coefficients
        assert self.length == n, f"`coefficients` must have length {self.length}"


def raised_cosine(t, symbol_duration, beta):
    """Raised-cosine pulse at times t (float32 array), evaluated in float32 like filter.py:394-405."""
    tt = np.abs(np.asarray(t, np.float32))
    with np.errstate(divide="ignore", invalid="ignore"):
        h = (1. / symbol_duration * np.sinc(tt / symbol_duration) * np.cos(np.pi * beta * tt / symbol_duration)
             / (1 - (2 * beta * tt / symbol_duration) ** 2)).astype(np.float32)
    if beta > 0:
        h[(tt - np.abs(symbol_duration / 2 / beta)) == 0] = np.pi / 4 / symbol_duration * np.sinc(1 / 2 / beta)
    return h


def root_raised_cosine(t, symbol_duration, beta):
    """Root-raised-cosine pulse at times t (float32 array), evaluated in float32 like filter.py:517-531."""
    tt = np.abs(np.asarray(t, np.float32))
    with np.errstate(divide="ignore", invalid="ignore"):
        h = (1 / symbol_duration / (np.pi * tt / symbol_duration * (1 - (4 * beta * tt / symbol_duration) ** 2))
             * (np.sin(np.pi * tt / symbol_duration * (1 - beta))
                + 4 * beta * tt / symbol_duration * np.cos(np.pi * tt / symbol_duration * (1 + beta)))).astype(np.float32)
    if beta > 0:
        h[(tt - np.abs(symbol_duration / 4 / beta)) == 0] = beta / symbol_duration / np.sqrt(2) * (
            (1 + 2 / np.pi) * np.sin(np.pi / 4 / beta) + (1 - 2 / np.pi) * np.cos(np.pi / 4 / beta))
    h[tt == 0] = 1 / symbol_duration * (1 + beta * (4 / np.pi - 1))
    return h
