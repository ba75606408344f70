"""OFDM channel estimation (mirror of /root/reference/src/sionna/phy/ofdm/channel_estimation.py:20-734):
``LSChannelEstimator`` with nearest-neighbour or (time-averaged) linear interpolation. The LMMSE interpolator of the
reference (:736-1855) is out of scope (SURVEY.md section 2)."""
from abc import abstractmethod
import numpy as np
import torch

from ..block import Block, Object
from ..._lib import lib, check, ptr, current_stream
from ..mapping import _broadcast_inner
from .resource_grid import ResourceGrid, RemoveNulledSubcarriers, gather_rows


class BaseChannelInterpolator(Object):
    """Interface: ``__call__(h_hat, err_var)`` with ``h_hat [batch, rx, rx_ant, tx, streams, num_pilots]`` ->
    ``[batch, rx, rx_ant, tx, streams, num_ofdm_symbols, num_effective_subcarriers]`` (:287-321)."""

    @abstractmethod
    def __call__(self, h_hat, err_var):
        pass


def _flat_ts(x, ts):
    """[..., tx, st, P] -> contiguous [B', ts, P] (B' = product of the leading dims)."""
    p = x.shape[-1]
    return x.reshape(-1, ts, p).contiguous()


class NearestNeighborInterpolator(BaseChannelInterpolator):
    """Every RE takes the estimate of the closest non-zero pilot in Manhattan (symbol, subcarrier) distance, first
    minimum in pilot order wins (:323-435)."""

    def __init__(self, pilot_pattern):
        super().__init__()
        assert pilot_pattern.num_pilot_symbols > 0, "The pilot pattern cannot be empty"
        mask = np.array(pilot_pattern.mask)
        mask_shape = mask.shape
        mask = mask.reshape([-1] + list(mask_shape[-2:]))
        pilots = np.reshape(pilot_pattern.pilots, [-1, pilot_pattern.pilots.shape[-1]])
        assert np.max(np.sum(np.abs(pilots) == 0, -1)) < pilots.shape[-1], \
            "Each pilot sequence must have at least one nonzero entry"
        s_, f_ = mask_shape[-2:]
        cols = np.arange(f_)[:, None]
        gather_ind = np.zeros((mask.shape[0], s_, f_), np.int32)
        for a in range(mask.shape[0]):
            i_p, j_p = np.where(mask[a])
            # zero pilots are never the nearest (the reference gives them a distance beyond any RE's), so only the
            # non-zero ones are candidates; one OFDM symbol at a time keeps the distance matrix at F x (non-zero pilots)
            nz = np.nonzero(np.abs(pilots[a]) > 0)[0]
            for s in range(s_):
                d = np.abs(s - i_p[nz])[None, :] + np.abs(cols - j_p[nz][None, :])
                gather_ind[a, s] = nz[np.argmin(d, axis=1)]
        self._gather_ind = gather_ind.reshape(mask.shape[0], s_ * f_)
        self._shape = mask_shape
        self._dev = None

    def _interpolate(self, x, floor0=False):
        tx, st, s_, f_ = self._shape
        ts = tx * st
        if self._dev is None or self._dev.device != x.device:
            self._dev = torch.from_numpy(self._gather_ind).to(x.device)
        lead = list(x.shape[:-3])
        xin = _flat_ts(x, ts)
        out = gather_rows(xin, self._dev, ts, s_ * f_, ts, xin.shape[-1])
        return out.reshape(lead + [tx, st, s_, f_])

    def __call__(self, h_hat, err_var):
        return self._interpolate(h_hat), self._interpolate(err_var)

    def interpolate_floored(self, h_hat, err_var):
        """Same, with the estimator's ``max(err_var, 0)`` (:171) applied inside the error-variance kernel."""
        return self._interpolate(h_hat), self._interpolate(err_var, floor0=True)


class LinearInterpolator(BaseChannelInterpolator):
    """Linear interpolation first along frequency on the pilot-carrying OFDM symbols (clamped linear extrapolation from
    the two nearest pilots), optional averaging over those symbols (``time_avg``), then along time (:437-734). The index
    tables follow :522-655."""

    def __init__(self, pilot_pattern, time_avg=False):
        super().__init__()
        assert pilot_pattern.num_pilot_symbols > 0, "The pilot pattern cannot be empty"
        self._time_avg = time_avg
        mask = np.array(pilot_pattern.mask)
        self._shape = mask.shape
        mask = mask.reshape([-1] + list(self._shape[-2:]))
        pilots = np.reshape(pilot_pattern.pilots, [-1, pilot_pattern.pilots.shape[-1]])
        assert np.max(np.sum(np.abs(pilots) == 0, -1)) < pilots.shape[-1], \
            "Each pilot sequence must have at least one nonzero entry"
        a_n, s_n, f_n = mask.shape
        z = np.zeros(mask.shape, pilots.dtype)
        for a in range(a_n):
            z[a][np.where(mask[a])] = pilots[a]
        x0 = np.zeros(mask.shape, np.int32)
        x1 = np.zeros(mask.shape, np.int32)
        nopil = np.sum(np.abs(z), axis=-1) == 0
        x0[nopil] = -1
        x1[nopil] = -1
        y0 = np.copy(x0)
        y1 = np.copy(x1)
        for a in range(a_n):
            pilot_count = 0
            pilot_ind = np.where(np.abs(pilots[a]))[0]
            for i in range(s_n):
                pio = np.where(np.abs(z[a][i]))[0]
                if len(pio) == 1:
                    x0[a, i] = pio[0]; x1[a, i] = pio[0]
                    y0[a, i] = pilot_ind[pilot_count]; y1[a, i] = pilot_ind[pilot_count]
                elif len(pio) >= 2:
                    k0, k1 = 0, 1
                    for j in range(f_n):
                        x0[a, i, j] = pio[k0]; x1[a, i, j] = pio[k1]
                        y0[a, i, j] = pilot_ind[pilot_count + k0]; y1[a, i, j] = pilot_ind[pilot_count + k1]
                        if j == pio[k1] and k1 < len(pio) - 1:
                            k0 = k1
                            k1 += 1
                pilot_count += len(pio)
        t0 = np.zeros((a_n, s_n), np.int32)
        t1 = np.zeros((a_n, s_n), np.int32)
        for a in range(a_n):
            ofdm_ind = np.where(np.sum(np.abs(z[a]), axis=-1))[0]
            if len(ofdm_ind) == 1:
                t0[a] = ofdm_ind[0]; t1[a] = ofdm_ind[0]
            elif len(ofdm_ind) >= 2:
                k0, k1 = 0, 1
                for i in range(s_n):
                    t0[a, i] = ofdm_ind[k0]; t1[a, i] = ofdm_ind[k1]
                    if i == ofdm_ind[k1] and k1 < len(ofdm_ind) - 1:
                        k0 = k1
                        k1 += 1
        npil = np.sum(np.sum(np.abs(z), axis=-1) > 0, axis=-1).astype(np.int32)
        self._tabs_np = [np.ascontiguousarray(t, np.int32) for t in (x0, x1, y0 + 1, y1 + 1, t0, t1, npil)]
        self._tabs = None

    def _interpolate(self, x, floor0=False):
        tx, st, s_, f_ = self._shape
        ts = tx * st
        if self._tabs is None or self._tabs[0].device != x.device:
            self._tabs = [torch.from_numpy(t).to(x.device) for t in self._tabs_np]
        lead = list(x.shape[:-3])
        cplx = x.is_complex()                                   # channel estimates: complex64, error variances: fp32
        xin = _flat_ts(x.to(torch.complex64 if cplx else torch.float32), ts)
        b, p = xin.shape[0], xin.shape[-1]
        out = torch.empty((b, ts, s_, f_), dtype=xin.dtype, device=x.device)
        t = self._tabs
        check(lib().sb_interp_lin(ptr(xin), ptr(t[0]), ptr(t[1]), ptr(t[2]), ptr(t[3]), ptr(t[4]), ptr(t[5]), ptr(t[6]),
                                  int(self._time_avg) | (2 if (floor0 and not cplx) else 0), ptr(out), b, ts, s_, f_, p,
                                  2 if cplx else 1, current_stream()),
              "sb_interp_lin")
        return out.reshape(lead + [tx, st, s_, f_])

    def __call__(self, h_hat, err_var):
        # the reference interpolates err_var as a complex tensor and keeps the real part (:729-732); same values in fp32
        return self._interpolate(h_hat), self._interpolate(err_var)

    def interpolate_floored(self, h_hat, err_var):
        """Same, with the estimator's ``max(err_var, 0)`` (:171) applied inside the error-variance kernel."""
        return self._interpolate(h_hat), self._interpolate(err_var, floor0=True)


class BaseChannelEstimator(Block):
    """Pilot gather + estimate at the pilots + interpolation over the grid (:20-173)."""

    def __init__(self, resource_grid, interpolation_type="nn", interpolator=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert isinstance(resource_grid, ResourceGrid), "You must provide a valid instance of ResourceGrid."
        self._resource_grid = resource_grid
        self._pilot_pattern = resource_grid.pilot_pattern
        self._remove_nulled_scs = RemoveNulledSubcarriers(resource_grid, precision=self.precision)
        assert interpolation_type in ["nn", "lin", "lin_time_avg", None], "Unsupported `interpolation_type`"
        self._interpolation_type = interpolation_type
        if interpolator is not None:
            assert isinstance(interpolator, BaseChannelInterpolator), \
                "`interpolator` must implement the BaseChannelInterpolator interface"
            self._interpol = interpolator
        elif interpolation_type == "nn":
            self._interpol = NearestNeighborInterpolator(self._pilot_pattern)
        elif interpolation_type == "lin":
            self._interpol = LinearInterpolator(self._pilot_pattern)
        elif interpolation_type == "lin_time_avg":
            self._interpol = LinearInterpolator(self._pilot_pattern, time_avg=True)
        num_pilot_symbols = self._pilot_pattern.num_pilot_symbols
        mask = self._pilot_pattern.mask.reshape(list(self._pilot_pattern.mask.shape[:2]) + [-1])
        # descending stable argsort: pilot REs first, in row-major order (:86-88)
        self._pilot_ind = np.argsort(-mask, axis=-1, kind="stable")[..., :num_pilot_symbols].astype(np.int32)

    @abstractmethod
    def estimate_at_pilot_locations(self, y_pilots, no):
        pass


class LSChannelEstimator(BaseChannelEstimator):
    """LSChannelEstimator(resource_grid, interpolation_type="nn", interpolator=None, precision=None)

    ``call(y, no)``: ``y [batch, num_rx, num_rx_ant, num_ofdm_symbols, fft_size]``, ``no`` [batch, num_rx, num_rx_ant] or
    its first n >= 0 dims -> ``h_hat`` / ``err_var`` ``[batch, num_rx, num_rx_ant, num_tx, num_streams_per_tx,
    num_ofdm_symbols, num_effective_subcarriers]``: ``h = y_p / p``, ``err_var = no / |p|^2`` at the pilots (0 where the
    pilot is 0), then interpolation (:175-285)."""

    def __init__(self, resource_grid, interpolation_type="nn", interpolator=None, precision=None, **kwargs):
        super().__init__(resource_grid, interpolation_type, interpolator, precision=precision, **kwargs)
        self._dev = None

    def estimate_at_pilot_locations(self, y_eff_flat, no):
        """y_eff_flat [B', L] (effective subcarriers, flattened grid), no broadcast -> h, err [B', ts, P]."""
        pp = self._pilot_pattern
        ts, p = pp.num_tx * pp.num_streams_per_tx, pp.num_pilot_symbols
        dev = y_eff_flat.device
        if self._dev is None or self._dev[0].device != dev:
            self._dev = (torch.from_numpy(self._pilot_ind.reshape(ts, p).copy()).to(dev),
                         torch.from_numpy(np.ascontiguousarray(pp.pilots.reshape(ts, p).astype(np.complex64))).to(dev))
        b, l = y_eff_flat.shape
        h = torch.empty((b, ts, p), dtype=torch.complex64, device=dev)
        err = torch.empty((b, ts, p), dtype=torch.float32, device=dev)
        no_t, inner = no
        check(lib().sb_ls_at_pilots(ptr(y_eff_flat), ptr(self._dev[0]), ptr(self._dev[1]), ptr(no_t), inner, ptr(h),
                                    ptr(err), b, ts, p, l, current_stream()), "sb_ls_at_pilots")
        return h, err

    def call(self, y, no):
        if self.precision != "single":
            raise NotImplementedError("LSChannelEstimator runs complex64 kernels only.")
        pp = self._pilot_pattern
        y_eff = self._remove_nulled_scs(y).to(torch.complex64)                  # [B, rx, ant, S, F]
        lead = list(y_eff.shape[:3])
        y_flat = y_eff.reshape(-1, y_eff.shape[-2] * y_eff.shape[-1]).contiguous()
        no_b = _broadcast_inner(no, lead, y_flat.device, torch.float32)          # element b' uses no[b' // inner]
        h, err = self.estimate_at_pilot_locations(y_flat, no_b)
        shp = lead + [pp.num_tx, pp.num_streams_per_tx, pp.num_pilot_symbols]
        h, err = h.reshape(shp), err.reshape(shp)
        if self._interpolation_type is not None:
            if isinstance(self._interpol, LinearInterpolator):
                h, err = self._interpol.interpolate_floored(h, err)            # max(err_var, 0) of :171 inside the kernel
            elif isinstance(self._interpol, NearestNeighborInterpolator):
                h, err = self._interpol(h, err)                                # a gather of no / |p|^2 >= 0: nothing to floor
            else:
                h, err = self._interpol(h, err)
                err = torch.clamp(err, min=0.0)                                  # :171 (user-supplied interpolator)
        return h, err
