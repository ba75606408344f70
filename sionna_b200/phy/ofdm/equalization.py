"""OFDM MIMO equalisation (mirror of /root/reference/src/sionna/phy/ofdm/equalization.py:17-462).

``LMMSEEqualizer`` runs ``sb_ofdm_lmmse`` (``whiten_interference=False``: ``sb_ofdm_equalize``), ``ZFEqualizer`` and
``MFEqualizer`` run ``sb_ofdm_equalize``: per resource element the receive vector, the desired / interfering channel
columns (``StreamManagement``), the noise and the channel-estimation error variances are read once, the covariance
``S = H_u H_u^H + diag(no) + diag(sum err_var)`` is assembled on chip, the LMMSE equaliser is applied and the soft symbols
of the data-carrying REs are written directly in the ``[batch, num_tx, num_streams, num_data_symbols]`` output layout. A
user-supplied equaliser callable is supported through ``OFDMEqualizer`` on the unfused route (explicit S tensor)."""
import numpy as np
import torch

from ..block import Block
from ..._lib import lib, check, ptr, current_stream
from .resource_grid import ResourceGrid, RemoveNulledSubcarriers


def _sm_tables(resource_grid, stream_management):
    """desired / undesired tx-stream indices per receiver, output stream row per (rx, k), data position per (stream, RE)."""
    rg, sm = resource_grid, stream_management
    txs = sm.num_tx * sm.num_streams_per_tx
    k = sm.num_streams_per_rx
    des = np.asarray(sm.detection_desired_ind).reshape(sm.num_rx, k) - np.arange(sm.num_rx)[:, None] * txs
    und = np.asarray(sm.detection_undesired_ind).reshape(sm.num_rx, -1) - np.arange(sm.num_rx)[:, None] * txs
    out_ts = np.argsort(np.asarray(sm.stream_ind), kind="stable").reshape(sm.num_rx, k)
    mask = rg.pilot_pattern.mask.reshape(txs, -1)
    nd = rg.pilot_pattern.num_data_symbols
    data_pos = np.full(mask.shape, -1, np.int32)
    for r in range(txs):
        data_ind = np.argsort(mask[r], kind="stable")[:nd]                 # equalization.py:104-107
        data_pos[r, data_ind] = np.arange(nd)
    return des.astype(np.int32), und.astype(np.int32), out_ts.astype(np.int32), data_pos


def _strides_for(t, full_shape):
    """Element strides of ``t`` viewed as broadcast to ``full_shape`` (0 on broadcast dims); t is made contiguous."""
    shp = [1] * (len(full_shape) - t.dim()) + list(t.shape)
    t = t.reshape(shp).contiguous()
    st = list(t.stride())
    return t, [0 if s == 1 and f != 1 else int(v) for s, f, v in zip(shp, full_shape, st)]


# equalisers with a fused kernel: name -> sb_ofdm_equalize's equaliser code ("lmmse" runs sb_ofdm_lmmse)
FUSED_EQUALIZERS = {"lmmse": 0, "lmmse-no-whitening": 1, "zf": 2, "mf": 3}


class OFDMEqualizer(Block):
    """OFDMEqualizer(equalizer, resource_grid, stream_management): wraps a MIMO equaliser ``(y, h, s) -> (x_hat, no_eff)``
    for OFDM (equalization.py:17-275). ``call(y, h_hat, err_var, no)`` returns ``x_hat`` / ``no_eff``
    ``[batch, num_tx, num_streams, num_data_symbols]``. A callable runs on the unfused route (explicit S tensor); a name
    of ``FUSED_EQUALIZERS`` runs its fused kernel."""

    def __init__(self, equalizer, resource_grid, stream_management, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert callable(equalizer) or equalizer in FUSED_EQUALIZERS
        assert isinstance(resource_grid, ResourceGrid)
        self._equalizer = equalizer
        self._resource_grid = resource_grid
        self._stream_management = stream_management
        self._removed_nulled_scs = RemoveNulledSubcarriers(resource_grid, precision=self.precision)
        self._tabs_np = _sm_tables(resource_grid, stream_management)
        self._tabs = None

    def _tables(self, dev):
        if self._tabs is None or self._tabs[0].device != dev:
            self._tabs = [torch.from_numpy(np.ascontiguousarray(t)).to(dev) for t in self._tabs_np]
        return self._tabs

    def call(self, y, h_hat, err_var, no):
        if self.precision != "single":
            raise NotImplementedError("OFDM equalisation runs complex64 kernels only.")
        if callable(self._equalizer):
            return self._unfused(*self._kernel_inputs(y, h_hat, err_var, no))
        sm = self._stream_management
        ptrs, sizes, _alive, nd = self._cabi_args(y, h_hat, err_var, no)
        shp = (sizes[0], sm.num_tx, sm.num_streams_per_tx, nd)
        x_hat = torch.zeros(shp, dtype=torch.complex64, device=self.device)
        no_eff = torch.zeros(shp, dtype=torch.float32, device=self.device)
        if self._equalizer == "lmmse":
            check(lib().sb_ofdm_lmmse(*ptrs, ptr(x_hat), ptr(no_eff), *sizes, current_stream()), "sb_ofdm_lmmse")
            return x_hat, no_eff
        check(lib().sb_ofdm_equalize(FUSED_EQUALIZERS[self._equalizer], *ptrs, ptr(x_hat), ptr(no_eff), *sizes,
                                     current_stream()), "sb_ofdm_equalize")
        return x_hat, no_eff

    def _cabi_args(self, y, h_hat, err_var, no):
        """The arguments ``sb_ofdm_lmmse`` and the OFDM detector entry points share: (pointers d_y ... d_data_pos,
        sizes batch ... num_data, the tensors and host stride arrays the caller keeps alive until the call returns,
        num_data)."""
        sm = self._stream_management
        y_eff, h, ev, ev_st, no_t, no_st = self._kernel_inputs(y, h_hat, err_var, no)
        b, rx, ant, s_, f_ = y_eff.shape
        des, und, out_ts, data_pos = self._tables(self.device)
        nd = self._resource_grid.pilot_pattern.num_data_symbols
        ev_arr = np.asarray(ev_st, np.int64)
        no_arr = np.asarray(no_st, np.int64)
        ptrs = [ptr(y_eff), ptr(h), ptr(ev), ptr(ev_arr), ptr(no_t), ptr(no_arr), ptr(des),
                ptr(und) if und.numel() else None, ptr(out_ts), ptr(data_pos)]
        sizes = [b, rx, ant, sm.num_tx * sm.num_streams_per_tx, s_, f_, sm.num_streams_per_rx,
                 sm.num_interfering_streams_per_rx, nd]
        return ptrs, sizes, (ev_arr, no_arr, y_eff, h, ev, no_t), nd

    def _kernel_inputs(self, y, h_hat, err_var, no):
        """The fused kernels' inputs: y [B, rx, ant, S, F] without nulled subcarriers, h [B, rx, ant, txs, S, F] and
        err_var / no as contiguous tensors with their broadcast strides (0 on broadcast dims)."""
        sm = self._stream_management
        dev = self.device
        y_eff = self._removed_nulled_scs(y).to(torch.complex64).contiguous()          # [B, rx, ant, S, F]
        b, rx, ant, s_, f_ = y_eff.shape
        txs = sm.num_tx * sm.num_streams_per_tx
        h = h_hat.to(device=dev, dtype=torch.complex64).reshape(b, rx, ant, txs, s_, f_).contiguous()
        full = [b, rx, ant, txs, s_, f_]
        ev = torch.as_tensor(err_var).to(device=dev, dtype=torch.float32)
        if ev.dim() == 7:
            ev = ev.reshape(list(ev.shape[:3]) + [ev.shape[3] * ev.shape[4]] + list(ev.shape[5:]))
        elif ev.dim() > 0:
            ev = ev.expand(torch.broadcast_shapes(tuple(ev.shape), tuple(h_hat.shape))).reshape(full)
        ev, ev_st = _strides_for(ev, full)
        no_t = torch.as_tensor(no).to(device=dev, dtype=torch.float32)
        no_t = no_t.reshape(list(no_t.shape) + [1] * (3 - no_t.dim()))                 # expand_to_rank(no, 3, -1)
        no_t, no_st = _strides_for(no_t, [b, rx, ant])
        return y_eff, h, ev, ev_st, no_t, no_st

    def _unfused(self, y_eff, h, ev, ev_st, no_t, no_st):
        """Generic equaliser callable: materialise y [B,rx,S,F,M], H [..,M,K], S [..,M,M] as the reference does
        (equalization.py:126-218), call it, then re-order streams and gather the data REs (:227-273)."""
        rg, sm = self._resource_grid, self._stream_management
        b, rx, ant, s_, f_ = y_eff.shape
        txs = sm.num_tx * sm.num_streams_per_tx
        des, und, out_ts, data_pos = self._tabs_np
        dev = y_eff.device
        y_dt = y_eff.permute(0, 1, 3, 4, 2)
        hp = h.permute(0, 1, 4, 5, 2, 3)                                                # [B, rx, S, F, M, txs]
        rows = torch.arange(rx, device=dev)[:, None]
        hd = torch.stack([hp[:, r][..., torch.as_tensor(des[r], device=dev)] for r in range(rx)], 1)
        s = torch.zeros((b, rx, s_, f_, ant, ant), dtype=torch.complex64, device=dev)
        if und.shape[1]:
            hu = torch.stack([hp[:, r][..., torch.as_tensor(und[r], device=dev)] for r in range(rx)], 1)
            s = hu @ hu.conj().transpose(-1, -2)
        ev_full = torch.as_strided(ev, [b, rx, ant, txs, s_, f_], ev_st).sum(3).permute(0, 1, 3, 4, 2)
        no_full = torch.as_strided(no_t, [b, rx, ant], no_st)[:, :, None, None, :]
        s = s + torch.diag_embed((ev_full + no_full).to(torch.complex64))
        x_hat, no_eff = self._equalizer(y_dt, hd, s)                                    # [B, rx, S, F, K]
        k = sm.num_streams_per_rx
        nd = rg.pilot_pattern.num_data_symbols
        xo = torch.zeros((b, txs, nd), dtype=x_hat.dtype, device=dev)
        no_o = torch.zeros((b, txs, nd), dtype=no_eff.dtype, device=dev)
        for r in range(rx):
            for kk in range(k):
                t = int(out_ts[r, kk])
                pos = torch.as_tensor(np.nonzero(data_pos[t] >= 0)[0], device=dev)
                xo[:, t] = x_hat[:, r, :, :, kk].reshape(b, -1)[:, pos]
                no_o[:, t] = no_eff[:, r, :, :, kk].reshape(b, -1)[:, pos]
        shp = (b, sm.num_tx, sm.num_streams_per_tx, nd)
        return xo.reshape(shp), no_o.reshape(shp)


class LMMSEEqualizer(OFDMEqualizer):
    """LMMSEEqualizer(resource_grid, stream_management, whiten_interference=True): LMMSE equalisation for OFDM MIMO
    (equalization.py:277-344); fused kernel ``sb_ofdm_lmmse``, or ``sb_ofdm_equalize`` with
    ``whiten_interference=False`` (``G = H^H (H H^H + S)^-1`` without whitening first)."""

    def __init__(self, resource_grid, stream_management, whiten_interference=True, precision=None, **kwargs):
        super().__init__("lmmse" if whiten_interference else "lmmse-no-whitening", resource_grid, stream_management,
                         precision=precision, **kwargs)


class ZFEqualizer(OFDMEqualizer):
    """ZFEqualizer(resource_grid, stream_management): ZF equalisation for OFDM MIMO (equalization.py:346-403,
    ``mimo.zf_equalizer`` per resource element); fused kernel ``sb_ofdm_equalize``."""

    def __init__(self, resource_grid, stream_management, precision=None, **kwargs):
        super().__init__("zf", resource_grid, stream_management, precision=precision, **kwargs)


class MFEqualizer(OFDMEqualizer):
    """MFEqualizer(resource_grid, stream_management): matched-filter equalisation for OFDM MIMO
    (equalization.py:405-462, ``mimo.mf_equalizer`` per resource element); fused kernel ``sb_ofdm_equalize``."""

    def __init__(self, resource_grid, stream_management, precision=None, **kwargs):
        super().__init__("mf", resource_grid, stream_management, precision=precision, **kwargs)
