"""OFDM transmit precoding (mirror of the reference's src/sionna/phy/ofdm/precoding.py:15-566) on ``sb_ofdm_precode``.

Per resource element and transmitter the kernel gathers the channel toward the transmitter's receivers
(``StreamManagement.precoding_ind``), computes the RZF / CBF / identity precoding matrix, scales its columns by
``sqrt(tx_power)``, precodes the symbols and forms the effective channel ``H_ij G_j`` toward every receiver i, so the
off-association entries carry the interference a receiver sees. Nulled subcarriers are removed from ``h_eff`` only.
Complex64 kernels; ``precision="double"`` falls back to them with a ``PrecisionWarning`` and returns complex128.
``PostEqualizationSINR`` is not provided."""
import numpy as np
import torch

from ..block import Block
from ..mimo.stream_management import StreamManagement
from ..._lib import lib, check, ptr, current_stream
from .resource_grid import ResourceGrid
from .equalization import _strides_for

_RZF, _CBF, _EYE = 0, 1, 2

_STREAM_MISMATCH = "The required number of streams per transmitter does not match the channel dimensions"


class _OFDMPrecoding(Block):
    """Resource grid and stream management of the precoding blocks, their device tables and the ``sb_ofdm_precode``
    call."""

    def __init__(self, resource_grid, stream_management, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert isinstance(resource_grid, ResourceGrid)
        assert isinstance(stream_management, StreamManagement)
        self._resource_grid = resource_grid
        self._stream_management = stream_management
        eff = np.asarray(resource_grid.effective_subcarrier_ind, np.int64)
        sc_pos = np.full(resource_grid.fft_size, -1, np.int32)
        sc_pos[eff] = np.arange(len(eff), dtype=np.int32)
        self._tabs_np = (np.ascontiguousarray(stream_management.precoding_ind, np.int32), sc_pos)
        self._tabs = None

    def _tables(self, dev):
        if self._tabs is None or self._tabs[0].device != dev:
            self._tabs = [torch.from_numpy(t).to(dev) for t in self._tabs_np]
        return self._tabs

    def _precode(self, kind, h, h_hat=None, x=None, alpha=None, alpha_left=False, tx_power=None, want_heff=True):
        """(x_precoded or None, h_eff or None). h, h_hat [B, RX, RA, TX, M, S, F]; x [B, TX, K, S, F]; alpha
        broadcast to [B, TX, S, F] aligned on the right (``alpha_left``: on the left); tx_power [B, TX, K, S, F] or its
        first n dimensions."""
        dev = self.device
        sm, rg = self._stream_management, self._resource_grid
        h = h.to(device=dev, dtype=torch.complex64).contiguous()
        b, rx, ra, tx, m, s_, f_ = h.shape
        if kind == _EYE:
            k = m
        else:
            k = sm.num_streams_per_tx
            if sm.num_rx_per_tx * ra != k:
                raise ValueError(_STREAM_MISMATCH)
        h_hat = h if h_hat is None else h_hat.to(device=dev, dtype=torch.complex64).contiguous()
        if x is not None:
            x = x.to(device=dev, dtype=torch.complex64).contiguous()
        pind, sc_pos = self._tables(dev)
        keep = []
        al = al_arr = None
        if kind == _RZF and alpha is not None:
            al = torch.as_tensor(alpha).to(device=dev, dtype=torch.float32)
            if alpha_left:                                          # expand_to_rank(alpha, 4, axis=-1)
                al = al.reshape(tuple(al.shape) + (1,) * (4 - al.dim()))
            al, st = _strides_for(al, [b, tx, s_, f_])
            al_arr = np.asarray(st, np.int64)
            keep += [al, al_arr]
        pw = pw_arr = None
        if tx_power is not None:                                    # expand_to_rank(tx_power, 6, axis=-1)
            pw = torch.as_tensor(tx_power).to(device=dev, dtype=torch.float32)
            pw = pw.reshape(tuple(pw.shape) + (1,) * (5 - pw.dim()))
            pw, st = _strides_for(pw, [b, tx, k, s_, f_])
            pw_arr = np.asarray(st, np.int64)
            keep += [pw, pw_arr]
        ne = rg.num_effective_subcarriers
        xp = torch.empty((b, tx, m, s_, f_), dtype=torch.complex64, device=dev) if x is not None else None
        heff = torch.empty((b, rx, ra, tx, k, s_, ne), dtype=torch.complex64, device=dev) if want_heff else None
        check(lib().sb_ofdm_precode(ptr(h_hat), ptr(h), ptr(pind), ptr(x), ptr(al), ptr(al_arr), ptr(pw), ptr(pw_arr),
                                    ptr(sc_pos), ptr(xp), ptr(heff), b, rx, ra, tx, m, k, s_, f_, ne, kind,
                                    current_stream()), "sb_ofdm_precode")
        return xp, heff


class RZFPrecoder(_OFDMPrecoding):
    """RZFPrecoder(resource_grid, stream_management, return_effective_channel=False): regularized zero-forcing
    precoding of OFDM resource grids (precoding.py:15-177).

    ``call(x, h, alpha=0.)``: x [B, num_tx, num_streams_per_tx, S, fft_size], h [B, num_rx, num_rx_ant, num_tx,
    num_tx_ant, S, fft_size], alpha broadcastable to [B, num_tx, S, fft_size] (aligned on the right,
    ``expand_to_rank(alpha, 4, axis=0)``). Returns x_precoded [B, num_tx, num_tx_ant, S, fft_size] and, if
    ``return_effective_channel``, h_eff [B, num_rx, num_rx_ant, num_tx, num_streams_per_tx, S,
    num_effective_subcarriers] toward every receiver."""

    def __init__(self, resource_grid, stream_management, return_effective_channel=False, precision=None, **kwargs):
        super().__init__(resource_grid, stream_management, precision=precision, **kwargs)
        self._return_effective_channel = return_effective_channel

    def call(self, x, h, alpha=0.):
        xp, heff = self._precode(_RZF, h, x=x, alpha=alpha, want_heff=self._return_effective_channel)
        return (xp, heff) if self._return_effective_channel else xp


class PrecodedChannel(_OFDMPrecoding):
    """PrecodedChannel(resource_grid, stream_management): base class of the blocks that return the effective channel
    after precoding, ``H_ij G_j diag(sqrt(p_j))`` for every receiver i and transmitter j (precoding.py:179-373).

    ``call(h, tx_power, h_hat=None, ...)``: h and h_hat [B, num_rx, num_rx_ant, num_tx, num_tx_ant, S, fft_size] (the
    precoder is computed from h_hat, h if None), tx_power [B, num_tx, num_streams_per_tx, S, fft_size] or its first n
    dimensions. Returns h_eff [B, num_rx, num_rx_ant, num_tx, num_streams_per_tx, S, num_effective_subcarriers]."""

    def call(self, h, tx_power, h_hat=None, **kwargs):
        raise NotImplementedError("PrecodedChannel is abstract: use RZFPrecodedChannel, CBFPrecodedChannel or "
                                  "EyePrecodedChannel")


class RZFPrecodedChannel(PrecodedChannel):
    """Effective channel after RZF precoding (precoding.py:375-446). ``alpha`` is broadcast to [B, num_tx, S,
    fft_size] aligned on the left (``expand_to_rank(alpha, 4, axis=-1)``)."""

    def call(self, h, tx_power, h_hat=None, alpha=0.):
        return self._precode(_RZF, h, h_hat=h_hat, alpha=alpha, alpha_left=True, tx_power=tx_power)[1]


class CBFPrecodedChannel(PrecodedChannel):
    """Effective channel after conjugate beamforming (precoding.py:448-510)."""

    def call(self, h, tx_power, h_hat=None):
        return self._precode(_CBF, h, h_hat=h_hat, tx_power=tx_power)[1]


class EyePrecodedChannel(PrecodedChannel):
    """Effective channel with the identity precoder and power allocation only, num_streams_per_tx = num_tx_ant
    (precoding.py:513-566)."""

    def call(self, h, tx_power):
        return self._precode(_EYE, h, tx_power=tx_power)[1]
