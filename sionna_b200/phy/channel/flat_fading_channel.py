"""Flat-fading MIMO channels (mirror of the reference's channel/flat_fading_channel.py:11-246) on ``sb_flat_fading``:
drawing h, correlating it (``KroneckerModel`` / ``PerColumnModel``), applying it to x and adding noise is one launch, and
h reaches global memory only when it is returned.

Randomness: the draw of h is ``complex_normal([batch_size, M, K])``'s, and the noise is ``AWGN``'s on ``y``, bit for bit
for the same (seed, offset) pairs. ``FlatFadingChannel`` takes the pairs in the order ``generate``, then ``apply`` (the
latter only with noise), so ``FlatFadingChannel(x, no)`` equals ``apply(x, generate(batch_size), no)`` bit for bit. A
user-defined ``SpatialCorrelation`` is called as the reference calls it: draw, correlate, apply."""
import torch

from ..block import Block
from ..config import config
from ..mapping import _broadcast_inner
from ..utils.misc import complex_normal
from ..._lib import lib, check, ptr, current_stream
from .spatial_correlation import KroneckerModel, PerColumnModel, factor_set


def flat_fading(lead, m, k, h=None, want_h=False, tx=None, rx=None, per_column=False, x=None, no=None):
    """One ``sb_flat_fading`` launch over the channel uses ``lead``: h from ``h [..., m, k]`` (broadcast against lead)
    or, if None, drawn; factors ``tx`` / ``rx`` = (contiguous tensor, stride); ``x [..., k]`` and ``no`` (AWGN's
    broadcasting on y). Returns (y [*lead, m] or None, h [*lead, m, k] or None)."""
    dev = config.device
    lead = tuple(int(v) for v in lead)
    num = int(torch.Size(lead).numel())
    h_in, h_stride, seed_h, off_h = None, 0, 0, 0
    if h is None:
        seed_h, off_h = config.next_philox()
    else:
        h_in, h_stride = factor_set(h, h.shape[:-2], lead, (m, k))
    h_out = torch.empty(lead + (m, k), dtype=torch.complex64, device=dev) if want_h else None
    xs, x_stride, y, no_t, inner, seed_n, off_n = None, 0, None, None, 1, 0, 0
    if x is not None:
        xs, x_stride = factor_set(x, x.shape[:-1], lead, (k,))
        y = torch.empty(lead + (m,), dtype=torch.complex64, device=dev)
        if no is not None:
            no_t, inner = _broadcast_inner(no, y.shape, dev, torch.float32)
            seed_n, off_n = config.next_philox()
    l_tx, tx_stride = tx if tx is not None else (None, 0)
    l_rx, rx_stride = rx if rx is not None else (None, 0)
    check(lib().sb_flat_fading(ptr(h_in), h_stride, seed_h, off_h, ptr(l_tx), tx_stride, ptr(l_rx), rx_stride,
                               int(per_column), ptr(h_out), ptr(xs), x_stride, ptr(no_t), inner, seed_n, off_n, ptr(y),
                               num, m, k, current_stream()), "sb_flat_fading")
    return y, h_out


def _fused(spatial_corr):
    """True if sb_flat_fading computes spatial_corr itself (None or one of the two models, not overridden)."""
    return spatial_corr is None or type(spatial_corr).__call__ in (KroneckerModel.__call__, PerColumnModel.__call__)


class GenerateFlatFadingChannel(Block):
    """GenerateFlatFadingChannel(num_tx_ant, num_rx_ant, spatial_corr=None, precision=None): ``__call__(batch_size)``
    -> ``h [batch_size, num_rx_ant, num_tx_ant]``, i.i.d. CN(0, 1) coefficients, then ``spatial_corr`` if set
    (flat_fading_channel.py:11-72)."""

    def __init__(self, num_tx_ant, num_rx_ant, spatial_corr=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._num_tx_ant = int(num_tx_ant)
        self._num_rx_ant = int(num_rx_ant)
        self.spatial_corr = spatial_corr

    @property
    def spatial_corr(self):
        """``SpatialCorrelation`` or None: get/set the spatial correlation to apply."""
        return self._spatial_corr

    @spatial_corr.setter
    def spatial_corr(self, value):
        self._spatial_corr = value

    def _plan(self, batch_size):
        """(fused, kernel factor arguments) for a draw of batch_size channels"""
        m, k, sc = self._num_rx_ant, self._num_tx_ant, self._spatial_corr
        if sc is None:
            return True, {}
        if not _fused(sc):
            return False, None
        lead, fac = sc.plan((int(batch_size),), m, k)
        return lead == (int(batch_size),), fac

    def call(self, batch_size):
        m, k = self._num_rx_ant, self._num_tx_ant
        fused, fac = self._plan(batch_size)
        if fused:
            return flat_fading((int(batch_size),), m, k, want_h=True, **fac)[1]
        return self._spatial_corr(complex_normal([int(batch_size), m, k]))


class ApplyFlatFadingChannel(Block):
    """ApplyFlatFadingChannel(precision=None): ``__call__(x, h, no=None)`` -> ``y = h x`` (+ CN(0, no) noise when
    ``no`` is given, broadcast as ``AWGN`` broadcasts it) with ``x [..., K]`` and ``h [..., M, K]`` whose leading
    dimensions broadcast against x's (flat_fading_channel.py:74-131)."""

    def call(self, x, h, no=None):
        m, k = h.shape[-2], h.shape[-1]
        if x.shape[-1] != k:
            raise ValueError(f"x has {x.shape[-1]} transmit antennas, h has {k}")
        lead = tuple(torch.broadcast_shapes(tuple(x.shape[:-1]), tuple(h.shape[:-2])))
        return flat_fading(lead, m, k, h=h, x=x, no=no)[0]


class FlatFadingChannel(Block):
    """FlatFadingChannel(num_tx_ant, num_rx_ant, spatial_corr=None, return_channel=False, precision=None):
    ``__call__(x, no=None)`` with ``x [batch_size, num_tx_ant]`` -> ``y [batch_size, num_rx_ant]``, or ``(y, h)``
    with ``return_channel`` (flat_fading_channel.py:133-246). Noise is added if and only if ``no`` is given; the
    reference's former ``add_awgn`` keyword is accepted and ignored. Without ``return_channel`` h is never written."""

    def __init__(self, num_tx_ant, num_rx_ant, spatial_corr=None, return_channel=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._num_tx_ant = int(num_tx_ant)
        self._num_rx_ant = int(num_rx_ant)
        self._return_channel = bool(return_channel)
        self._gen_chn = GenerateFlatFadingChannel(num_tx_ant, num_rx_ant, spatial_corr, precision=precision)
        self._app_chn = ApplyFlatFadingChannel(precision=precision)

    @property
    def spatial_corr(self):
        """``SpatialCorrelation`` or None: get/set the spatial correlation to apply."""
        return self._gen_chn.spatial_corr

    @spatial_corr.setter
    def spatial_corr(self, value):
        self._gen_chn.spatial_corr = value

    @property
    def generate(self):
        """The internal ``GenerateFlatFadingChannel``."""
        return self._gen_chn

    @property
    def apply(self):
        """The internal ``ApplyFlatFadingChannel``."""
        return self._app_chn

    def call(self, x, no=None):
        b = int(x.shape[0])
        fused, fac = self._gen_chn._plan(b) if x.dim() == 2 else (False, None)
        if fused:
            y, h = flat_fading((b,), self._num_rx_ant, self._num_tx_ant, want_h=self._return_channel, x=x, no=no,
                               **fac)
        else:
            h = self._gen_chn(b)
            y = self._app_chn(x, h, no)
        return (y, h) if self._return_channel else y
