"""OFDM MIMO detection (mirror of /root/reference/src/sionna/phy/ofdm/detection.py:20-1173): ``LinearDetector``
= fused LMMSE / ZF / MF equalisation (``sb_ofdm_lmmse``, ``sb_ofdm_equalize``) + demapping with the per-symbol
effective noise variance (``sb_demap``, or ``sb_symbol_demap`` for symbol outputs);
``MaximumLikelihoodDetector`` / ``MaximumLikelihoodDetectorWithPrior`` = fused covariance assembly + ML detection
(``sb_ofdm_ml``); ``KBestDetector``, ``EPDetector`` and ``MMSEPICDetector`` = the same assembly + K-Best, EP or
MMSE-PIC detection (``sb_ofdm_kbest``, ``sb_ofdm_ep``, ``sb_ofdm_mmse_pic``)."""
import torch

from ..._lib import lib, check, ptr, current_stream
from ..block import Block
from ..mapping import Constellation, Demapper, SymbolDemapper
from ..mimo.detection import (llrs_to_symbol_logits, ml_check_limits, detector_workspace, detector_out,
                              KBestDetector as _MimoKBest, EPDetector as _MimoEP, MMSEPICDetector as _MimoPIC,
                              iterative_check_limits, EP_MAX_POINTS, PIC_MAX_POINTS)
from .equalization import LMMSEEqualizer, ZFEqualizer, MFEqualizer, OFDMEqualizer


class LinearDetector(Block):
    """LinearDetector(equalizer, output, demapping_method, resource_grid, stream_management, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    OFDM equaliser followed by a demapper (detection.py:740-847; PUSCH default ``("lmmse","bit","maxlog")``):
    ``equalizer`` ``"lmmse"`` / ``"zf"`` / ``"mf"`` runs the fused ``LMMSEEqualizer`` / ``ZFEqualizer`` /
    ``MFEqualizer``, a callable ``(y, h, s) -> (x_hat, no_eff)`` runs through ``OFDMEqualizer``'s unfused route.
    ``call(y, h_hat, err_var, no)`` -> LLRs / hard bits ``[batch, num_tx, num_streams,
    num_data_symbols*num_bits_per_symbol]`` (``output="bit"``), logits ``[batch, num_tx, num_streams, num_data_symbols,
    num_points]`` or int32 indices ``[batch, num_tx, num_streams, num_data_symbols]`` (``output="symbol"``)."""

    def __init__(self, equalizer, output, demapping_method, resource_grid, stream_management, constellation_type=None,
                 num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        # same argument checks and error types as the reference (mimo/detection.py:103-115)
        assert not isinstance(equalizer, str) or equalizer in ["lmmse", "zf", "mf"], "Unknown equalizer."
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        if equalizer == "lmmse":
            self._equalizer = LMMSEEqualizer(resource_grid, stream_management, precision=precision)
        elif equalizer == "zf":
            self._equalizer = ZFEqualizer(resource_grid, stream_management, precision=precision)
        elif equalizer == "mf":
            self._equalizer = MFEqualizer(resource_grid, stream_management, precision=precision)
        else:
            self._equalizer = OFDMEqualizer(equalizer, resource_grid, stream_management, precision=precision)
        if output == "bit":
            self._demapper = Demapper(demapping_method, constellation=self._constellation, hard_out=hard_out,
                                      precision=precision)
        else:
            self._demapper = SymbolDemapper(constellation=self._constellation, hard_out=hard_out, precision=precision)

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
        dev, sm = self.device, self._eq._stream_management
        ptrs, sizes, _alive, nd = self._eq._cabi_args(y, h_hat, err_var, no)
        b, rx, _, txs, s_, f_ = sizes[:6]
        m = self._constellation.num_bits_per_symbol
        npts = 2 ** m
        pr = None
        if prior is not None:
            pr = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if self._output == "bit":
                pr = llrs_to_symbol_logits(pr.reshape(b, txs, nd, m), m)
            pr = pr.reshape(b, txs, nd, npts).contiguous()
        out = detector_out(self._output, self._hard_out, m, [b, sm.num_tx, sm.num_streams_per_tx, nd], dev).zero_()
        pts = self._constellation().to(device=dev, dtype=torch.complex64).contiguous()
        ws = detector_workspace(lib().sb_ml_workspace_bytes(b * rx * s_ * f_, sm.num_streams_per_rx), dev)
        check(lib().sb_ofdm_ml(*ptrs, ptr(pr), ptr(pts), ptr(out), ptr(ws), ws.numel(), *sizes, npts, self._method,
                               int(self._output == "symbol"), int(self._hard_out), current_stream()), "sb_ofdm_ml")
        return out.flatten(-2) if self._output == "bit" else out


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
        dev, det, sm = self.device, self._detector, self._eq._stream_management
        ptrs, sizes, _alive, nd = self._eq._cabi_args(y, h_hat, err_var, no)
        b, rx, ant, _, s_, f_ = sizes[:6]
        if ant < sm.num_streams_per_rx:
            raise AssertionError("The number of receive antennas cannot be smaller than the number of streams")
        m = det._num_bits_out
        out = detector_out(self._output, det._hard_out, m, [b, sm.num_tx, sm.num_streams_per_tx, nd], dev).zero_()
        pts, kk, real_rep, symbol, hard, clip = det._kernel_args(dev)
        ws = detector_workspace(lib().sb_kbest_workspace_bytes(b * rx * s_ * f_, sm.num_streams_per_rx, real_rep), dev)
        check(lib().sb_ofdm_kbest(*ptrs, ptr(pts), ptr(out), ptr(ws), ws.numel(), *sizes, 2 ** m, kk, real_rep, symbol,
                                  hard, clip, current_stream()), "sb_ofdm_kbest")
        return out.flatten(-2) if self._output == "bit" else out


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
        ptrs, sizes, _alive, nd = self._eq._cabi_args(y, h_hat, err_var, no)
        lev, npts, l, beta, symbol, hard = det._kernel_args(dev)
        out = detector_out(det._output, det._hard_out, det._num_bits_per_symbol,
                           [sizes[0], sm.num_tx, sm.num_streams_per_tx, nd], dev).zero_()
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
        ptrs, sizes, _alive, nd = self._eq._cabi_args(y, h_hat, err_var, no)
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
