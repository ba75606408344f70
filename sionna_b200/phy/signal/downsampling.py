"""Downsampling (mirror of /root/reference/src/sionna/phy/signal/downsampling.py) on ``sb_gather_rows``."""
import numpy as np

from ..block import Block
from .upsampling import gather_last, IndexCache


class Downsampling(Block):
    """Downsampling(samples_per_symbol, offset=0, num_symbols=None, axis=-1, precision=None)

    Keeps one out of ``samples_per_symbol`` samples of ``x`` [..., n, ...] along ``axis``, starting at ``offset``, and
    at most ``num_symbols`` of them (downsampling.py:9-79). The kept indices are Python's own slice
    ``range(n)[offset::samples_per_symbol][:num_symbols]``, so negative offsets and offsets >= n (an empty result)
    behave as in the reference; the length is ceil((n - offset) / samples_per_symbol) before ``num_symbols`` (the
    reference's docstring says floor, its slicing gives ceil). Exact in float32, float64, complex64, complex128 and the
    32- and 64-bit integers; unlike the reference, bool and 8- or 16-bit integers raise ``NotImplementedError``."""
    _native_double = True

    def __init__(self, samples_per_symbol, offset=0, num_symbols=None, axis=-1, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._samples_per_symbol = samples_per_symbol
        self._offset = offset
        self._num_symbols = num_symbols
        self._axis = axis
        self._index = IndexCache(self._make_index)

    def _make_index(self, n):
        idx = np.arange(n)[self._offset::self._samples_per_symbol]
        return idx if self._num_symbols is None else idx[:self._num_symbols]

    def call(self, inputs):
        return gather_last(inputs, self._axis, self._index.get(inputs.shape[self._axis], inputs.device))
