"""OFDM MIMO detection (mirror of /root/reference/src/sionna/phy/ofdm/detection.py:20-1173): ``LinearDetector``
= fused LMMSE equalisation (``sb_ofdm_lmmse``) + demapping with the per-symbol effective noise variance (``sb_demap``);
``MaximumLikelihoodDetector`` / ``MaximumLikelihoodDetectorWithPrior`` = fused covariance assembly + ML detection
(``sb_ofdm_ml``); ``KBestDetector``, ``EPDetector`` and ``MMSEPICDetector`` = the same assembly + K-Best, EP or
MMSE-PIC detection (``sb_ofdm_kbest``, ``sb_ofdm_ep``, ``sb_ofdm_mmse_pic``)."""
import numpy as np
import torch

from ..._lib import lib, check, ptr, current_stream
from ..block import Block
from ..mapping import Constellation, Demapper
from ..mimo.detection import (llrs_to_symbol_logits, ml_check_limits, ml_workspace, KBestDetector as _MimoKBest,
                              kbest_workspace, EPDetector as _MimoEP, MMSEPICDetector as _MimoPIC,
                              iterative_check_limits, EP_MAX_POINTS, PIC_MAX_POINTS)
from .equalization import LMMSEEqualizer, OFDMEqualizer


class LinearDetector(Block):
    """LinearDetector(equalizer, output, demapping_method, resource_grid, stream_management, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    ``call(y, h_hat, err_var, no)`` -> LLRs ``[batch, num_tx, num_streams, num_data_symbols*num_bits_per_symbol]``
    (``output="bit"``); ``equalizer="lmmse"`` (detection.py:740-847; PUSCH default ``("lmmse","bit","maxlog")``)."""

    def __init__(self, equalizer, output, demapping_method, resource_grid, stream_management, constellation_type=None,
                 num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        # same argument checks and error types as the reference (mimo/detection.py:103-115)
        assert not isinstance(equalizer, str) or equalizer in ["lmmse", "zf", "mf"], "Unknown equalizer."
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        if equalizer != "lmmse":
            raise NotImplementedError(f"equalizer={equalizer!r}: only 'lmmse' has a fused OFDM kernel here.")
        if output != "bit":
            raise NotImplementedError("output='symbol' (SymbolDemapper) is not provided; use output='bit'.")
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        self._equalizer = LMMSEEqualizer(resource_grid, stream_management, precision=precision)
        self._demapper = Demapper(demapping_method, constellation=self._constellation, hard_out=hard_out,
                                  precision=precision)

    def call(self, y, h_hat, err_var, no):
        x_hat, no_eff = self._equalizer(y, h_hat, err_var, no)
        return self._demapper(x_hat, no_eff)


class MaximumLikelihoodDetector(Block):
    """MaximumLikelihoodDetector(output, demapping_method, resource_grid, stream_management, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    ML detection for OFDM MIMO (detection.py:524-647) on the fused ``sb_ofdm_ml`` kernel: the interference-plus-noise
    covariance of every resource element is assembled on chip from ``OFDMEqualizer``'s stream tables, then every
    candidate vector of the receiver's streams is scored as in ``mimo.MaximumLikelihoodDetector``.
    ``call(y, h_hat, err_var, no)`` -> ``[batch, num_tx, num_streams, num_data_symbols*num_bits_per_symbol]`` LLRs / hard
    bits (``output="bit"``), ``[batch, num_tx, num_streams, num_data_symbols, num_points]`` logits or
    ``[batch, num_tx, num_streams, num_data_symbols]`` int32 indices (``output="symbol"``)."""

    def __init__(self, output, demapping_method, resource_grid, stream_management, constellation_type=None,
                 num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        self._output = output
        self._method = 0 if demapping_method == "app" else 1
        self._hard_out = bool(hard_out)
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        ml_check_limits(stream_management.num_streams_per_rx, self._constellation.num_points)
        self._eq = OFDMEqualizer("lmmse", resource_grid, stream_management, precision=precision)

    @property
    def constellation(self):
        return self._constellation

    def call(self, y, h_hat, err_var, no):
        return self._detect(y, h_hat, None, err_var, no)

    def _detect(self, y, h_hat, prior, err_var, no):
        eq = self._eq
        rg, sm = eq._resource_grid, eq._stream_management
        dev = self.device
        y_eff, h, ev, ev_st, no_t, no_st = eq._kernel_inputs(y, h_hat, err_var, no)
        b, rx, ant, s_, f_ = y_eff.shape
        txs = sm.num_tx * sm.num_streams_per_tx
        des, und, out_ts, data_pos = eq._tables(dev)
        nd = rg.pilot_pattern.num_data_symbols
        m = self._constellation.num_bits_per_symbol
        npts = 2 ** m
        pr = None
        if prior is not None:
            pr = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if self._output == "bit":
                pr = llrs_to_symbol_logits(pr.reshape(b, txs, nd, m), m)
            pr = pr.reshape(b, txs, nd, npts).contiguous()
        shp = [b, sm.num_tx, sm.num_streams_per_tx]
        if self._output == "bit":
            out = torch.zeros(shp + [nd * m], dtype=torch.float32, device=dev)
        elif self._hard_out:
            out = torch.zeros(shp + [nd], dtype=torch.int32, device=dev)
        else:
            out = torch.zeros(shp + [nd, npts], dtype=torch.float32, device=dev)
        pts = self._constellation().to(device=dev, dtype=torch.complex64).contiguous()
        ev_arr = np.asarray(ev_st, np.int64)                    # host stride arrays: alive until the call returns
        no_arr = np.asarray(no_st, np.int64)
        ws = ml_workspace(b * rx * s_ * f_, sm.num_streams_per_rx, dev)
        check(lib().sb_ofdm_ml(ptr(y_eff), ptr(h), ptr(ev), ptr(ev_arr), ptr(no_t), ptr(no_arr), ptr(des),
                               ptr(und) if und.numel() else None, ptr(out_ts), ptr(data_pos), ptr(pr), ptr(pts), ptr(out),
                               ptr(ws), ws.numel(), b, rx, ant, txs, s_, f_,
                               sm.num_streams_per_rx, sm.num_interfering_streams_per_rx, nd, npts, self._method,
                               int(self._output == "symbol"), int(self._hard_out), current_stream()), "sb_ofdm_ml")
        return out


class MaximumLikelihoodDetectorWithPrior(MaximumLikelihoodDetector):
    """MaximumLikelihoodDetectorWithPrior(output, demapping_method, resource_grid, stream_management, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    ``MaximumLikelihoodDetector`` with prior knowledge of the transmitted signals (detection.py:650-738):
    ``call(y, h_hat, prior, err_var, no)``, ``prior`` = bit LLRs ``[batch, num_tx, num_streams,
    num_data_symbols*num_bits_per_symbol]`` (``output="bit"``) or point logits ``[batch, num_tx, num_streams,
    num_data_symbols, num_points]`` (``output="symbol"``). Stream k of a receiver takes the prior of the transmitted
    stream it detects."""

    def call(self, y, h_hat, prior, err_var, no):
        return self._detect(y, h_hat, prior, err_var, no)


class KBestDetector(Block):
    """KBestDetector(output, num_streams, k, resource_grid, stream_management, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, use_real_rep=False, list2llr=None, precision=None)

    K-Best detection for OFDM MIMO (detection.py:849-967) on the fused ``sb_ofdm_kbest`` kernel: the
    interference-plus-noise covariance of every resource element is assembled on chip from ``OFDMEqualizer``'s stream
    tables, then the receiver's streams are detected as in ``mimo.KBestDetector`` (same arguments, checks and limits).
    ``call(y, h_hat, err_var, no)`` -> ``[batch, num_tx, num_streams, num_data_symbols*num_bits_per_symbol]`` LLRs / hard
    bits (``output="bit"``) or ``[batch, num_tx, num_streams, num_data_symbols]`` int32 indices (``output="symbol"``,
    ``hard_out=True``). ``num_streams`` must equal ``stream_management.num_streams_per_rx`` (ValueError)."""

    def __init__(self, output, num_streams, k, resource_grid, stream_management, constellation_type=None,
                 num_bits_per_symbol=None, constellation=None, hard_out=False, use_real_rep=False, list2llr=None,
                 precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if int(num_streams) != stream_management.num_streams_per_rx:
            raise ValueError(f"KBestDetector: num_streams = {num_streams}, but every receiver detects "
                             f"stream_management.num_streams_per_rx = {stream_management.num_streams_per_rx} streams")
        self._detector = _MimoKBest(output, num_streams, k, constellation_type=constellation_type,
                                    num_bits_per_symbol=num_bits_per_symbol, constellation=constellation,
                                    hard_out=hard_out, use_real_rep=use_real_rep, list2llr=list2llr,
                                    precision=precision)
        self._output = output
        self._eq = OFDMEqualizer("lmmse", resource_grid, stream_management, precision=precision)

    @property
    def list2llr(self):
        """The wrapped detector's ``List2LLRSimple`` (soft bit outputs)."""
        return self._detector.list2llr

    def call(self, y, h_hat, err_var, no):
        eq, det = self._eq, self._detector
        rg, sm = eq._resource_grid, eq._stream_management
        dev = self.device
        y_eff, h, ev, ev_st, no_t, no_st = eq._kernel_inputs(y, h_hat, err_var, no)
        b, rx, ant, s_, f_ = y_eff.shape
        if ant < sm.num_streams_per_rx:
            raise AssertionError("The number of receive antennas cannot be smaller than the number of streams")
        txs = sm.num_tx * sm.num_streams_per_tx
        des, und, out_ts, data_pos = eq._tables(dev)
        nd = rg.pilot_pattern.num_data_symbols
        m = det._num_bits_out
        shp = [b, sm.num_tx, sm.num_streams_per_tx]
        if self._output == "bit":
            out = torch.zeros(shp + [nd * m], dtype=torch.float32, device=dev)
        else:
            out = torch.zeros(shp + [nd], dtype=torch.int32, device=dev)
        pts, kk, real_rep, symbol, hard, clip = det._kernel_args(dev)
        ev_arr = np.asarray(ev_st, np.int64)                    # host stride arrays: alive until the call returns
        no_arr = np.asarray(no_st, np.int64)
        ws = kbest_workspace(b * rx * s_ * f_, sm.num_streams_per_rx, real_rep, dev)
        check(lib().sb_ofdm_kbest(ptr(y_eff), ptr(h), ptr(ev), ptr(ev_arr), ptr(no_t), ptr(no_arr), ptr(des),
                                  ptr(und) if und.numel() else None, ptr(out_ts), ptr(data_pos), ptr(pts), ptr(out),
                                  ptr(ws), ws.numel(), b, rx, ant, txs, s_, f_, sm.num_streams_per_rx,
                                  sm.num_interfering_streams_per_rx, nd, 2 ** m, kk, real_rep, symbol, hard, clip,
                                  current_stream()), "sb_ofdm_kbest")
        return out


def _ofdm_kernel_inputs(eq, y, h_hat, err_var, no, dev):
    """(leading C-ABI arguments up to d_data_pos, [batch .. num_data] sizes, host stride arrays kept alive by the
    caller, num_data) of the OFDM detector entry points."""
    rg, sm = eq._resource_grid, eq._stream_management
    y_eff, h, ev, ev_st, no_t, no_st = eq._kernel_inputs(y, h_hat, err_var, no)
    b, rx, ant, s_, f_ = y_eff.shape
    txs = sm.num_tx * sm.num_streams_per_tx
    des, und, out_ts, data_pos = eq._tables(dev)
    nd = rg.pilot_pattern.num_data_symbols
    ev_arr = np.asarray(ev_st, np.int64)
    no_arr = np.asarray(no_st, np.int64)
    ptrs = [ptr(y_eff), ptr(h), ptr(ev), ptr(ev_arr), ptr(no_t), ptr(no_arr), ptr(des),
            ptr(und) if und.numel() else None, ptr(out_ts), ptr(data_pos)]
    sizes = [b, rx, ant, txs, s_, f_, sm.num_streams_per_rx, sm.num_interfering_streams_per_rx, nd]
    return ptrs, sizes, (ev_arr, no_arr, y_eff, h, ev, no_t), nd


class EPDetector(Block):
    """EPDetector(output, resource_grid, stream_management, num_bits_per_symbol=None, hard_out=False, l=10, beta=0.9, precision=None)

    EP detection for OFDM MIMO (detection.py:969-1060) on the fused ``sb_ofdm_ep`` kernel: the interference-plus-noise
    covariance of every resource element is assembled on chip from ``OFDMEqualizer``'s stream tables, then the
    receiver's streams are detected as in ``mimo.EPDetector`` (same arguments, checks and limits).
    ``call(y, h_hat, err_var, no)`` -> ``[batch, num_tx, num_streams, num_data_symbols*num_bits_per_symbol]`` LLRs / hard
    bits (``output="bit"``), ``[batch, num_tx, num_streams, num_data_symbols, num_points]`` logits or
    ``[batch, num_tx, num_streams, num_data_symbols]`` int32 indices (``output="symbol"``)."""

    def __init__(self, output, resource_grid, stream_management, num_bits_per_symbol=None, hard_out=False, l=10,
                 beta=0.9, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._detector = _MimoEP(output, num_bits_per_symbol, hard_out=hard_out, l=l, beta=beta, precision=precision)
        iterative_check_limits("EPDetector", stream_management.num_streams_per_rx, 2 ** int(num_bits_per_symbol),
                               EP_MAX_POINTS)
        self._eq = OFDMEqualizer("lmmse", resource_grid, stream_management, precision=precision)

    def call(self, y, h_hat, err_var, no):
        dev, det, sm = self.device, self._detector, self._eq._stream_management
        ptrs, sizes, _alive, nd = _ofdm_kernel_inputs(self._eq, y, h_hat, err_var, no, dev)
        lev, npts, l, beta, symbol, hard = det._kernel_args(dev)
        out = det._out([sizes[0], sm.num_tx, sm.num_streams_per_tx, nd], dev).zero_()
        check(lib().sb_ofdm_ep(*ptrs, ptr(lev), ptr(out), *sizes, npts, l, beta, symbol, hard, current_stream()),
              "sb_ofdm_ep")
        return out.flatten(-2) if det._output == "bit" else out


class MMSEPICDetector(Block):
    """MMSEPICDetector(output, demapping_method, resource_grid, stream_management, num_iter=1, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    MMSE-PIC detection for OFDM MIMO (detection.py:1062-1173) on the fused ``sb_ofdm_mmse_pic`` kernel: the
    interference-plus-noise covariance of every resource element is assembled on chip from ``OFDMEqualizer``'s stream
    tables, then the receiver's streams are detected as in ``mimo.MMSEPICDetector`` (same arguments, checks and
    limits). ``call(y, h_hat, prior, err_var, no)``, ``prior`` in ``MaximumLikelihoodDetectorWithPrior``'s layout: bit
    LLRs ``[batch, num_tx, num_streams, num_data_symbols*num_bits_per_symbol]`` (``output="bit"``) or point logits
    ``[batch, num_tx, num_streams, num_data_symbols, num_points]`` (``output="symbol"``); stream k of a receiver takes
    the prior of the transmitted stream it detects, streams without data at an element a zero prior. Outputs in the
    layouts of ``MaximumLikelihoodDetector``: extrinsic LLRs / hard bits, logits or int32 indices."""

    def __init__(self, output, demapping_method, resource_grid, stream_management, num_iter=1, constellation_type=None,
                 num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._detector = _MimoPIC(output, demapping_method, num_iter, constellation_type=constellation_type,
                                  num_bits_per_symbol=num_bits_per_symbol, constellation=constellation,
                                  hard_out=hard_out, precision=precision)
        iterative_check_limits("MMSEPICDetector", stream_management.num_streams_per_rx,
                               self._detector.constellation.num_points, PIC_MAX_POINTS)
        self._eq = OFDMEqualizer("lmmse", resource_grid, stream_management, precision=precision)

    @property
    def constellation(self):
        return self._detector.constellation

    def call(self, y, h_hat, prior, err_var, no):
        dev, det, sm = self.device, self._detector, self._eq._stream_management
        ptrs, sizes, _alive, nd = _ofdm_kernel_inputs(self._eq, y, h_hat, err_var, no, dev)
        m = det.constellation.num_bits_per_symbol
        shp = [sizes[0], sm.num_tx, sm.num_streams_per_tx, nd]
        pr = torch.as_tensor(prior)
        pr = det._prior_llrs(pr.reshape(shp + ([m] if det._output == "bit" else [2 ** m])), shp, dev)
        out = torch.zeros(shp + [m], dtype=torch.float32, device=dev)
        pts, npts, num_iter, method, hard = det._kernel_args(dev)
        check(lib().sb_ofdm_mmse_pic(*ptrs, ptr(pr), ptr(pts), ptr(out), *sizes, npts, num_iter, method, hard,
                                     current_stream()), "sb_ofdm_mmse_pic")
        out = det._finish(out)
        return out.flatten(-2) if det._output == "bit" else out
