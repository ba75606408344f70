"""Window functions (mirror of /root/reference/src/sionna/phy/signal/window.py) on ``sb_scale_last``
(``csrc/signal.cu``). Coefficients are built on the host in float64 NumPy from the input length, as in the reference,
and cast to the block's precision; the product runs natively in float32 or float64."""
import numpy as np
import torch

from ..block import Block
from ..._lib import lib, check, ptr, current_stream


class Window(Block):
    """Abstract window function, applied by element-wise multiplication along the last dimension (window.py:12-163).

    Parameters: ``normalize`` (bool, default False): scale the window to unit average power per coefficient,
    ``w / sqrt(mean(w^2))``; ``precision``. Input: ``x`` [..., N] real or complex, N equal to ``length``. Output: same
    shape and dtype as ``x``. ``show`` is not provided (no plotting). No autograd."""
    _native_double = True

    def __init__(self, normalize=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert isinstance(normalize, bool), "normalize must be bool"
        self._normalize = normalize
        self._coefficients = None

    @property
    def coefficients(self):
        """[N], float: Set/get raw window coefficients (before normalization)."""
        return self._coefficients

    @coefficients.setter
    def coefficients(self, v):
        self._coefficients = self._cast_or_check_precision(v)

    @property
    def length(self):
        """int: Window length in number of samples."""
        return self.coefficients.shape[0]

    @property
    def normalize(self):
        """bool: If True, the window is normalized to have unit average power per coefficient."""
        return self._normalize

    def show(self, samples_per_symbol, domain="time", scale="lin"):
        """Not provided: this package has no plotting (window.py:84-143)."""
        raise NotImplementedError("Window.show: plotting is not provided")

    def call(self, x):
        w = self.coefficients
        if w.is_complex():
            raise TypeError("window coefficients must be real")
        if x.dtype not in (self.rdtype, self.cdtype):
            raise TypeError(f"Window: x must be a real or complex floating-point tensor, not {x.dtype}")
        if w.requires_grad or x.requires_grad:
            raise NotImplementedError("Window: gradients are not supported (the signal kernels have no backward)")
        n = x.shape[-1]
        if n != w.shape[0]:
            raise ValueError(f"the last dimension of x ({n}) must equal the window length ({w.shape[0]})")
        x = x.contiguous()
        w = w.contiguous()
        y = torch.empty_like(x)
        rows = x.numel() // n if n else 0
        check(lib().sb_scale_last(ptr(x), int(x.is_complex()), ptr(w), ptr(y), int(self.precision == "double"), rows,
                                  n, int(self._normalize), current_stream()), "sb_scale_last")
        return y


class CustomWindow(Window):
    """Window with user-given coefficients [N], real (window.py:165-209)."""

    def __init__(self, coefficients, normalize=False, precision=None, **kwargs):
        super().__init__(normalize=normalize, precision=precision, **kwargs)
        self.coefficients = coefficients


class HannWindow(Window):
    """Hann window ``w_n = sin^2(pi n / N)``, 0 <= n <= N - 1 (window.py:211-262)."""

    def build(self, input_shape):
        length = input_shape[-1]
        n = np.arange(length)
        self.coefficients = np.sin(np.pi * n / length) ** 2


class HammingWindow(Window):
    """Hamming window ``w_n = a0 - (1 - a0) cos(2 pi n / N)``, a0 = 25/46 (window.py:264-317)."""

    def build(self, input_shape):
        length = input_shape[-1]
        n = np.arange(length)
        a0 = 25. / 46.
        self.coefficients = a0 - (1. - a0) * np.cos(2. * np.pi * n / length)


class BlackmanWindow(Window):
    """Blackman window ``w_n = a0 - a1 cos(2 pi n / N) + a2 cos(4 pi n / N)``, a0 = 7938/18608, a1 = 9240/18608,
    a2 = 1430/18608 (window.py:319-373)."""

    def build(self, input_shape):
        length = input_shape[-1]
        n = np.arange(length)
        a0, a1, a2 = 7938. / 18608., 9240. / 18608., 1430. / 18608.
        self.coefficients = a0 - a1 * np.cos(2. * np.pi * n / length) + a2 * np.cos(4. * np.pi * n / length)
