"""OFDM resource grid and (de)mapping (mirror of /root/reference/src/sionna/phy/ofdm/resource_grid.py)."""
import numpy as np
import torch

from ..block import Block, Object
from ..._lib import lib, check, ptr, current_stream
from .pilot_pattern import PilotPattern, EmptyPilotPattern, KroneckerPilotPattern


def gather_rows(x, idx_dev, rows, cols_out, in_rows, cols_in):
    """out[b, r, j] = x[b, (0 | r), idx[r, j]] through ``sb_gather_rows``; x is [batch, in_rows, cols_in] (float32 or
    complex64, contiguous; float64 / complex128 are copied bit for bit as 2 / 4 words); returns [batch, rows, cols_out]."""
    if x.dtype not in (torch.float32, torch.complex64, torch.float64, torch.complex128):
        raise NotImplementedError(f"gather_rows: unsupported dtype {x.dtype}")
    words = x.element_size() // 4
    x = x.contiguous()
    batch = x.numel() // (in_rows * cols_in)
    out = torch.empty((batch, rows, cols_out), dtype=x.dtype, device=x.device)
    check(lib().sb_gather_rows(ptr(x), ptr(idx_dev), ptr(out), batch, rows, cols_out, in_rows, cols_in, words,
                               current_stream()), "sb_gather_rows")
    return out


class ResourceGrid(Object):
    """ResourceGrid(num_ofdm_symbols, fft_size, subcarrier_spacing, num_tx=1, num_streams_per_tx=1, cyclic_prefix_length=0, num_guard_carriers=(0,0), dc_null=False, pilot_pattern=None, pilot_ofdm_symbol_indices=None, precision=None)

    OFDM resource grid spanning ``num_ofdm_symbols`` x ``fft_size`` resource elements with guard carriers, optional DC
    null and a pilot pattern (resource_grid.py:15-392). RE types: 0 data, 1 pilot, 2 guard, 3 DC."""

    def __init__(self, num_ofdm_symbols, fft_size, subcarrier_spacing, num_tx=1, num_streams_per_tx=1,
                 cyclic_prefix_length=0, num_guard_carriers=(0, 0), dc_null=False, pilot_pattern=None,
                 pilot_ofdm_symbol_indices=None, precision=None):
        super().__init__(precision=precision)
        self._num_ofdm_symbols = num_ofdm_symbols
        self._fft_size = fft_size
        self._subcarrier_spacing = subcarrier_spacing
        self._cyclic_prefix_length = int(cyclic_prefix_length)
        self._num_tx = num_tx
        self._num_streams_per_tx = num_streams_per_tx
        self._num_guard_carriers = np.array(num_guard_carriers)
        self._dc_null = dc_null
        self._pilot_ofdm_symbol_indices = pilot_ofdm_symbol_indices
        self.pilot_pattern = pilot_pattern
        self._check_settings()

    @property
    def cyclic_prefix_length(self):
        return self._cyclic_prefix_length

    @property
    def num_tx(self):
        return self._num_tx

    @property
    def num_streams_per_tx(self):
        return self._num_streams_per_tx

    @property
    def num_ofdm_symbols(self):
        return self._num_ofdm_symbols

    @property
    def num_resource_elements(self):
        return self._fft_size * self._num_ofdm_symbols

    @property
    def num_effective_subcarriers(self):
        return int(self._fft_size - self._dc_null - np.sum(self._num_guard_carriers))

    @property
    def effective_subcarrier_ind(self):
        num_gc = self._num_guard_carriers
        sc_ind = np.arange(num_gc[0], self.fft_size - num_gc[1])
        if self.dc_null:
            sc_ind = np.delete(sc_ind, self.dc_ind - num_gc[0])
        return sc_ind

    @property
    def num_data_symbols(self):
        return int(self.num_effective_subcarriers * self._num_ofdm_symbols - self.num_pilot_symbols)

    @property
    def num_pilot_symbols(self):
        return self.pilot_pattern.num_pilot_symbols

    @property
    def num_zero_symbols(self):
        return int((self._fft_size - self.num_effective_subcarriers) * self._num_ofdm_symbols)

    @property
    def num_guard_carriers(self):
        return self._num_guard_carriers

    @property
    def dc_ind(self):
        return int(self._fft_size / 2 - (self._fft_size % 2 == 1) / 2)

    @property
    def fft_size(self):
        return self._fft_size

    @property
    def subcarrier_spacing(self):
        return self._subcarrier_spacing

    @property
    def ofdm_symbol_duration(self):
        return (1. + self.cyclic_prefix_length / self.fft_size) / self.subcarrier_spacing

    @property
    def bandwidth(self):
        return self.fft_size * self.subcarrier_spacing

    @property
    def num_time_samples(self):
        return (self.fft_size + self.cyclic_prefix_length) * self._num_ofdm_symbols

    @property
    def dc_null(self):
        return self._dc_null

    @property
    def pilot_pattern(self):
        return self._pilot_pattern

    @pilot_pattern.setter
    def pilot_pattern(self, value):
        if value is None or (isinstance(value, str) and value == "empty"):
            value = EmptyPilotPattern(self._num_tx, self._num_streams_per_tx, self._num_ofdm_symbols,
                                      self.num_effective_subcarriers, precision=self.precision)
        elif isinstance(value, PilotPattern):
            pass
        elif isinstance(value, str):
            assert value in ["kronecker", "empty"], "Unknown pilot pattern"
            assert self._pilot_ofdm_symbol_indices is not None, "You must provide pilot_ofdm_symbol_indices."
            value = KroneckerPilotPattern(self, self._pilot_ofdm_symbol_indices, precision=self.precision)
        else:
            raise ValueError("Unsupported pilot_pattern")
        self._pilot_pattern = value

    def _check_settings(self):
        assert self._num_ofdm_symbols > 0, "`num_ofdm_symbols` must be positive`."
        assert self._fft_size > 0, "`fft_size` must be positive`."
        assert self._cyclic_prefix_length >= 0, "`cyclic_prefix_length must be nonnegative."
        assert self._cyclic_prefix_length <= self._fft_size, "`cyclic_prefix_length cannot be longer than `fft_size`."
        assert self._num_tx > 0, "`num_tx` must be positive`."
        assert self._num_streams_per_tx > 0, "`num_streams_per_tx` must be positive`."
        assert len(self._num_guard_carriers) == 2, "`num_guard_carriers` must have two elements."
        assert np.all(np.greater_equal(self._num_guard_carriers, 0)), "`num_guard_carriers` must have nonnegative entries."
        assert np.sum(self._num_guard_carriers) <= self._fft_size - self._dc_null, \
            "Total number of guardcarriers cannot be larger than `fft_size`."
        return True

    def build_type_grid(self):
        """[num_tx, num_streams_per_tx, num_ofdm_symbols, fft_size] int32 RE types (resource_grid.py:283-311)."""
        shape = [self._num_tx, self._num_streams_per_tx, self._num_ofdm_symbols]
        gc_l = 2 * np.ones(shape + [self._num_guard_carriers[0]], np.int32)
        gc_r = 2 * np.ones(shape + [self._num_guard_carriers[1]], np.int32)
        dc = 3 * np.ones(shape + [int(self._dc_null)], np.int32)
        mask = self.pilot_pattern.mask
        split_ind = self.dc_ind - self._num_guard_carriers[0]
        return np.concatenate([gc_l, mask[..., :split_ind], dc, mask[..., split_ind:], gc_r], -1).astype(np.int32)


class ResourceGridMapper(Block):
    """ResourceGridMapper(resource_grid): ``[batch, num_tx, num_streams_per_tx, num_data_symbols]`` data symbols ->
    ``[batch, num_tx, num_streams_per_tx, num_ofdm_symbols, fft_size]`` grid with pilots, data written in row-major
    (symbol, subcarrier) order over the type-0 REs (resource_grid.py:313-412)."""

    def __init__(self, resource_grid, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._resource_grid = rg = resource_grid
        t = rg.build_type_grid().reshape(rg.num_tx * rg.num_streams_per_tx, -1)
        m = np.full(t.shape, -1, np.int32)
        for r in range(t.shape[0]):
            d = np.nonzero(t[r] == 0)[0]
            m[r, d] = np.arange(len(d))
            p = np.nonzero(t[r] == 1)[0]
            m[r, p] = -(np.arange(len(p)) + 2)
        self._map = m
        self._dev = None

    def call(self, inputs):
        rg = self._resource_grid
        if self.precision != "single":
            raise NotImplementedError("sb_rg_map is a complex64 kernel.")
        dev = self.device
        if self._dev is None or self._dev[0].device != dev:
            pil = np.ascontiguousarray(rg.pilot_pattern.pilots.reshape(self._map.shape[0], -1))
            self._dev = (torch.from_numpy(self._map).to(dev), torch.from_numpy(pil).to(dev) if pil.size else None)
        x = inputs.to(device=dev, dtype=torch.complex64).contiguous()
        b = x.shape[0]
        ts, g = self._map.shape
        out = torch.empty((b, rg.num_tx, rg.num_streams_per_tx, rg.num_ofdm_symbols, rg.fft_size),
                          dtype=torch.complex64, device=dev)
        check(lib().sb_rg_map(ptr(x), ptr(self._dev[1]), ptr(self._dev[0]), ptr(out), b, ts, g, x.shape[-1],
                              rg.num_pilot_symbols, current_stream()), "sb_rg_map")
        return out


class RemoveNulledSubcarriers(Block):
    """Drops guard and DC subcarriers: ``[..., fft_size] -> [..., num_effective_subcarriers]`` (resource_grid.py:522-553)."""

    _native_double = True                   # a bit copy: float64 / complex128 pass through unrounded

    def __init__(self, resource_grid, precision=None, **kwargs):
        self._sc_ind = np.asarray(resource_grid.effective_subcarrier_ind, np.int32)
        self._fft_size = resource_grid.fft_size
        super().__init__(precision=precision, **kwargs)
        self._idx = None

    def call(self, inputs):
        dev = self.device
        if self._idx is None or self._idx.device != dev:
            self._idx = torch.from_numpy(self._sc_ind[None, :].copy()).to(dev)
        x = inputs.to(dev).contiguous()
        n = len(self._sc_ind)
        out = gather_rows(x, self._idx, 1, n, 1, self._fft_size)
        return out.reshape(list(x.shape[:-1]) + [n])


class ResourceGridDemapper(Block):
    """ResourceGridDemapper(resource_grid, stream_management): extracts the data REs of every stream from
    ``[batch, num_rx, num_streams_per_rx, num_ofdm_symbols, fft_size(, data_dim)]`` ->
    ``[batch, num_tx, num_streams_per_tx, num_data_symbols(, data_dim)]`` (resource_grid.py:414-520)."""

    _native_double = True                   # a bit copy: float64 / complex128 pass through unrounded

    def __init__(self, resource_grid, stream_management, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._stream_management = sm = stream_management
        self._resource_grid = rg = resource_grid
        mask = rg.pilot_pattern.mask.reshape(rg.num_tx * rg.num_streams_per_tx, -1)
        nd = rg.pilot_pattern.num_data_symbols
        eff = np.asarray(rg.effective_subcarrier_ind)
        f_eff = len(eff)
        grid = rg.num_ofdm_symbols * rg.fft_size
        idx = np.zeros((mask.shape[0], nd), np.int64)
        for r in range(mask.shape[0]):
            data_ind = np.argsort(mask[r], kind="stable")[:nd]            # ascending: non-pilot REs first (:461-465)
            sym, sc = data_ind // f_eff, data_ind % f_eff
            idx[r] = sm.stream_ind[r] * grid + sym * rg.fft_size + eff[sc]
        self._idx_np = idx
        self._idx = {}

    def call(self, y):
        rg, sm = self._resource_grid, self._stream_management
        dev = self.device
        has_dd = y.dim() == 6
        dd = y.shape[-1] if has_dd else 1
        key = (dd, dev)
        if key not in self._idx:
            idx = self._idx_np[:, :, None] * dd + np.arange(dd)[None, None, :]
            self._idx[key] = torch.from_numpy(idx.reshape(idx.shape[0], -1).astype(np.int32)).to(dev)
        x = y.to(dev).contiguous()
        b = x.shape[0]
        rows, cols = self._idx[key].shape
        total_in = sm.num_rx * sm.num_streams_per_rx * rg.num_ofdm_symbols * rg.fft_size * dd
        out = gather_rows(x, self._idx[key], rows, cols, 1, total_in)
        shp = [b, rg.num_tx, rg.num_streams_per_tx, rg.pilot_pattern.num_data_symbols]
        return out.reshape(shp + ([dd] if has_dd else []))
