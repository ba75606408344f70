"""Upsampling by zero insertion (mirror of /root/reference/src/sionna/phy/signal/upsampling.py) on ``sb_gather_rows``:
output sample j takes input sample j / sps where sps divides j and is 0 (index -1) elsewhere, a bit copy of 4-, 8- and
16-byte elements (float32, float64, complex64, complex128 and the 32- and 64-bit integers)."""
import numpy as np
import torch

from ..block import Block
from ..ofdm.resource_grid import gather_rows


_WORDS = {4: torch.float32, 8: torch.float64}      # integer elements are copied as floats of their size, bit for bit


def gather_last(x, axis, idx_dev):
    """x with the ``axis`` dimension replaced by x[..., idx] (idx: int32 device tensor, -1 gives 0), through
    ``sb_gather_rows``. Elements of 1 or 2 bytes (bool, 8- and 16-bit integers) raise ``NotImplementedError``."""
    dt = x.dtype
    if dt.is_floating_point or dt.is_complex:
        as_dt = dt
    elif x.element_size() in _WORDS:
        as_dt = _WORDS[x.element_size()]
    else:
        raise NotImplementedError(f"up/downsampling copies 4-, 8- or 16-byte elements; {dt} is not supported")
    x = x.movedim(axis, -1)
    n = x.shape[-1]
    lead = tuple(x.shape[:-1])
    y = gather_rows(x.reshape(-1, 1, n).contiguous().view(as_dt), idx_dev, 1, idx_dev.shape[0], 1, n)
    return y.view(dt).reshape(lead + (idx_dev.shape[0],)).movedim(-1, axis)


class IndexCache:
    """The device copy of a block's gather index for each input length and device it has seen, built once."""

    def __init__(self, make):
        self._make, self._tables = make, {}

    def get(self, n, device):
        key = (n, device)
        if key not in self._tables:
            self._tables[key] = torch.as_tensor(np.asarray(self._make(n), np.int32), device=device)
        return self._tables[key]


class Upsampling(Block):
    """Upsampling(samples_per_symbol, axis=-1, precision=None)

    Upsamples ``x`` [..., n, ...] along ``axis`` by inserting ``samples_per_symbol - 1`` zeros after every sample
    (upsampling.py:10-72): output [..., n * samples_per_symbol, ...], same dtype. Exact in float32, float64,
    complex64, complex128 and the 32- and 64-bit integers; unlike the reference, bool and 8- or 16-bit integers raise
    ``NotImplementedError``."""
    _native_double = True

    def __init__(self, samples_per_symbol, axis=-1, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._samples_per_symbol = samples_per_symbol
        self._axis = axis
        self._index = IndexCache(self._make_index)

    def _make_index(self, n):
        idx = np.full(n * self._samples_per_symbol, -1, np.int32)
        idx[::self._samples_per_symbol] = np.arange(n)
        return idx

    def call(self, inputs):
        return gather_last(inputs, self._axis, self._index.get(inputs.shape[self._axis], inputs.device))
