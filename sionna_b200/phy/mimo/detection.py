"""MIMO detection (mirror of /root/reference/src/sionna/phy/mimo/detection.py:24-1643): linear, maximum-likelihood,
K-Best, EP and MMSE-PIC."""
import warnings

import numpy as np
import torch

from ..._lib import lib, check, ptr, current_stream
from ..block import Block
from ..mapping import Constellation, Demapper, SymbolDemapper, pam
from .equalization import lmmse_equalizer, zf_equalizer, mf_equalizer


class LinearDetector(Block):
    """LinearDetector(equalizer, output, demapping_method, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    Equaliser followed by a demapper (detection.py:87-143): ``call(y, h, s)`` -> LLRs / hard bits
    ``[..., K, num_bits_per_symbol]`` (``output="bit"``, ``Demapper``) or logits ``[..., K, num_points]`` / int32
    indices ``[..., K]`` (``output="symbol"``, ``SymbolDemapper``). ``equalizer`` is ``"lmmse"``, ``"zf"``, ``"mf"``
    or a callable ``(y, h, s) -> (x_hat, no_eff)``."""

    def __init__(self, equalizer, output, demapping_method, constellation_type=None, num_bits_per_symbol=None,
                 constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._output = output
        self._hard_out = hard_out
        # same argument checks and error types as the reference (detection.py:103-115)
        if isinstance(equalizer, str):
            assert equalizer in ["lmmse", "zf", "mf"], "Unknown equalizer."
            equalizer = {"lmmse": lmmse_equalizer, "zf": zf_equalizer, "mf": mf_equalizer}[equalizer]
        self._equalizer = equalizer
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        if output == "bit":
            self._demapper = Demapper(demapping_method, constellation=self._constellation, hard_out=hard_out,
                                      precision=precision)
        else:
            self._demapper = SymbolDemapper(constellation=self._constellation, hard_out=hard_out, precision=precision)

    def call(self, y, h, s):
        x_hat, no_eff = self._equalizer(y, h, s)
        z = self._demapper(x_hat, no_eff)
        if self._output == "symbol":
            return z
        m = self._constellation.num_bits_per_symbol
        return z.reshape(list(x_hat.shape) + [m])


ML_MAX_STREAMS = 8
ML_MAX_CANDIDATES = 65536
ML_MAX_POINTS = 1024


def ml_check_limits(num_streams, num_points):
    """ValueError unless 1 <= num_streams <= 8, num_points <= 1024 and num_points ** num_streams <= 65536 (the limits of
    the ``sb_mimo_ml`` / ``sb_ofdm_ml`` kernels)."""
    if not 1 <= int(num_streams) <= ML_MAX_STREAMS:
        raise ValueError(f"MaximumLikelihoodDetector: {num_streams} streams, supported are 1 ... {ML_MAX_STREAMS}")
    if num_points > ML_MAX_POINTS or num_points ** int(num_streams) > ML_MAX_CANDIDATES:
        raise ValueError(f"MaximumLikelihoodDetector: {num_streams} streams of a {num_points}-point constellation are "
                         f"{num_points ** int(num_streams)} candidate vectors; supported are at most "
                         f"{ML_MAX_CANDIDATES} and constellations of at most {ML_MAX_POINTS} points")


def detector_workspace(nbytes, device):
    """Workspace of ``nbytes`` for the ML and K-Best entry points (``sb_ml_workspace_bytes`` /
    ``sb_kbest_workspace_bytes``) from PyTorch's caching allocator."""
    return torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device=device)


def detector_out(output, hard_out, num_bits_per_symbol, shape, device):
    """Uninitialised detector output: LLRs / hard bits ``[*shape, m]`` (``output="bit"``), int32 symbol indices
    ``[*shape]`` (``output="symbol"`` with ``hard_out``) or symbol logits ``[*shape, 2**m]``."""
    m = num_bits_per_symbol
    if output == "bit":
        return torch.empty(shape + [m], dtype=torch.float32, device=device)
    if hard_out:
        return torch.empty(shape, dtype=torch.int32, device=device)
    return torch.empty(shape + [2 ** m], dtype=torch.float32, device=device)


def llrs_to_symbol_logits(llrs, num_bits_per_symbol):
    """LLRs2SymbolLogits (mapping.py:1045-1059): ``[..., m]`` bit LLRs -> ``[..., 2**m]`` point logits
    ``sum_i log_sigmoid(a_ci * llr_i)``, a_ci = +1 / -1 for label bit i (MSB first) of point c equal to 1 / 0."""
    m = num_bits_per_symbol
    a = 2.0 * ((torch.arange(2 ** m, device=llrs.device)[:, None] >> torch.arange(m - 1, -1, -1, device=llrs.device)) & 1) - 1.0
    return torch.nn.functional.logsigmoid(llrs[..., None, :] * a.to(llrs.dtype)).sum(-1)


def _dense_inputs(y, h, s, k, dev):
    """(y [B, M], h [B, M, K], s [B, M, M] complex64 contiguous, batch shape, M, number of problems) after broadcasting
    the batch dimensions of the three inputs."""
    h = torch.as_tensor(h).to(device=dev, dtype=torch.complex64)
    mm = h.shape[-2]
    if h.shape[-1] != k:
        raise ValueError(f"h must have num_streams = {k} as last dimension")
    batch = torch.broadcast_shapes(tuple(torch.as_tensor(y).shape[:-1]), tuple(h.shape[:-2]),
                                   tuple(torch.as_tensor(s).shape[:-2]))
    y = torch.as_tensor(y).to(device=dev, dtype=torch.complex64).expand(list(batch) + [mm]).contiguous()
    h = h.expand(list(batch) + [mm, k]).contiguous()
    s = torch.as_tensor(s).to(device=dev, dtype=torch.complex64).expand(list(batch) + [mm, mm]).contiguous()
    return y, h, s, list(batch), mm, int(np.prod(batch)) if len(batch) else 1


class MaximumLikelihoodDetector(Block):
    """MaximumLikelihoodDetector(output, demapping_method, num_streams, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    MIMO maximum-likelihood detection (detection.py:145-537) on the fused ``sb_mimo_ml`` kernel: whitening with S,
    every one of the |C|^K candidate vectors scored on chip, logsumexp (``"app"``) or max (``"maxlog"``) per stream and
    point. ``call(y [..., M], h [..., M, K], s [..., M, M], prior=None)`` -> LLRs / hard bits ``[..., K, m]``
    (``output="bit"``; ``prior``: bit LLRs ``[..., K, m]``) or logits ``[..., K, |C|]`` / int32 indices ``[..., K]``
    (``output="symbol"``; ``prior``: point logits ``[..., K, |C|]``). Limits: K <= 8, |C| <= 1024, |C|^K <= 65536
    (ValueError otherwise)."""

    def __init__(self, output, demapping_method, num_streams, constellation_type=None, num_bits_per_symbol=None,
                 constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        self._output = output
        self._method = 0 if demapping_method == "app" else 1
        self._hard_out = bool(hard_out)
        self._num_streams = int(num_streams)
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        ml_check_limits(self._num_streams, self._constellation.num_points)

    @property
    def constellation(self):
        return self._constellation

    def call(self, y, h, s, prior=None):
        dev = self.device
        k, m = self._num_streams, self._constellation.num_bits_per_symbol
        npts = 2 ** m
        y, h, s, batch, mm, num = _dense_inputs(y, h, s, k, dev)
        pr = None
        if prior is not None:
            pr = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if self._output == "bit":
                pr = llrs_to_symbol_logits(pr, m)
            pr = pr.expand(batch + [k, npts]).contiguous()
        out = detector_out(self._output, self._hard_out, m, batch + [k], dev)
        pts = self._constellation().to(device=dev, dtype=torch.complex64).contiguous()
        ws = detector_workspace(lib().sb_ml_workspace_bytes(num, k), dev)
        check(lib().sb_mimo_ml(ptr(y), ptr(h), ptr(s), ptr(pr), ptr(pts), ptr(out), ptr(ws), ws.numel(), num, mm, k, npts,
                               self._method, int(self._output == "symbol"), int(self._hard_out), current_stream()),
              "sb_mimo_ml")
        return out


KB_MAX_LAYERS = 16
KB_MAX_K = 256
KB_MAX_POINTS = 256
KB_MAX_CHILDREN = 16384


def kbest_check_limits(num_layers, k, num_points):
    """ValueError unless the detection domain (``num_layers`` = streams, or twice that in the real-valued
    representation, of ``num_points`` points) is within the limits of ``sb_mimo_kbest`` / ``sb_ofdm_kbest``: at most 16
    layers, k <= 256, 256 points and k * num_points <= 16384."""
    if num_layers > KB_MAX_LAYERS:
        raise ValueError(f"KBestDetector: {num_layers} detection layers, supported are at most {KB_MAX_LAYERS} "
                         f"(16 streams, or 8 with use_real_rep=True)")
    if k > KB_MAX_K or num_points > KB_MAX_POINTS or k * num_points > KB_MAX_CHILDREN:
        raise ValueError(f"KBestDetector: k = {k} paths of a {num_points}-point detection constellation; supported are "
                         f"k <= {KB_MAX_K}, at most {KB_MAX_POINTS} points and k * points <= {KB_MAX_CHILDREN}")


class List2LLR(Block):
    """Base class of the rules that turn a K-Best candidate list into LLRs (mimo/utils.py:365-418). Only
    ``List2LLRSimple`` is provided: it runs inside the K-Best kernel, which never materialises the list."""

    def call(self, y, r, dists, path_inds, path_syms):
        raise NotImplementedError("List2LLR rules run inside KBestDetector's kernel; only List2LLRSimple is provided")


class List2LLRSimple(List2LLR):
    """List2LLRSimple(num_bits_per_symbol, llr_clip_val=20.0, precision=None)

    LLR(k, i) = min metric over the paths whose bit i of stream k is 0 minus the min over those where it is 1 (an empty
    set counts as +inf), clipped to +-``llr_clip_val`` (mimo/utils.py:420-577; ``np.inf`` disables the clipping). Used
    as ``KBestDetector``'s ``list2llr``, which reads ``llr_clip_val`` at every call."""

    def __init__(self, num_bits_per_symbol, llr_clip_val=20.0, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._num_bits_per_symbol = int(num_bits_per_symbol)
        self.llr_clip_val = llr_clip_val

    @property
    def llr_clip_val(self):
        """Absolute value to which the LLRs are clipped."""
        return self._llr_clip_val

    @llr_clip_val.setter
    def llr_clip_val(self, value):
        self._llr_clip_val = value


class KBestDetector(Block):
    """KBestDetector(output, num_streams, k, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, use_real_rep=False, list2llr=None, precision=None)

    MIMO K-Best detection (detection.py:539-1037) on the fused ``sb_mimo_kbest`` kernel: whitening with S, columns
    sorted by descending norm, QR, then a breadth-first tree search from the last sorted stream that keeps the k paths
    with the smallest metrics per layer (ties: lower candidate index first, as ``tf.math.top_k``). ``use_real_rep``
    detects the real-valued equivalent channel (QAM only) on PAM layers. ``call(y [..., M], h [..., M, num_streams],
    s [..., M, M])`` -> LLRs / hard bits ``[..., num_streams, num_bits_per_symbol]`` (``output="bit"``; LLRs from
    ``List2LLRSimple``) or int32 symbol indices ``[..., num_streams]`` (``output="symbol"``, needs ``hard_out=True``).
    ``k`` is clipped to the number of candidate vectors with a warning. Limits, in the detection domain: at most 16
    layers (streams, or twice the streams with ``use_real_rep``), k <= 256, at most 256 points and k * points <= 16384
    (ValueError otherwise)."""

    def __init__(self, output, num_streams, k, constellation_type=None, num_bits_per_symbol=None, constellation=None,
                 hard_out=False, use_real_rep=False, list2llr=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        # same argument checks and error types as the reference (detection.py:691-800)
        assert output in ("bit", "symbol"), "Unknown output"
        err_msg = "You must provide either constellation or constellation_type and num_bits_per_symbol."
        if constellation is None:
            assert constellation_type is not None and num_bits_per_symbol is not None, err_msg
        else:
            assert constellation_type is None and num_bits_per_symbol is None, err_msg
            assert constellation.precision == self.precision, "Constellation has wrong precision."
        self._output = output
        self._hard_out = bool(hard_out)
        self._use_real_rep = bool(use_real_rep)
        self._num_tx_streams = int(num_streams)
        if self._use_real_rep:
            err_msg = "Only QAM can be used for the real-valued representation"
            if constellation_type is not None:
                assert constellation_type == "qam", err_msg
            else:
                assert constellation.constellation_type == "qam", err_msg
            self._num_streams = 2 * self._num_tx_streams
            n = (constellation.num_bits_per_symbol if num_bits_per_symbol is None else num_bits_per_symbol) // 2
            self._num_bits_per_symbol = n
            c = pam(n, normalize=False, precision=precision)       # PAM scaled to energy 0.5, as the reference builds it
            c = c / (np.std(c) * np.sqrt(2)).astype(c.dtype)
            self._constellation = np.real(c)
            self._num_bits_out = 2 * n
        else:
            self._num_streams = self._num_tx_streams
            c = Constellation.check_or_create(constellation_type=constellation_type,
                                              num_bits_per_symbol=num_bits_per_symbol, constellation=constellation,
                                              precision=precision)
            self._constellation = c().cpu().numpy()
            self._num_bits_per_symbol = c.num_bits_per_symbol
            self._num_bits_out = c.num_bits_per_symbol
        self._num_symbols = self._constellation.shape[0]
        self._k = min(int(k), self._num_symbols ** self._num_streams)
        if self._k < k:
            warnings.warn(f"KBestDetector: The provided value of k={k} is larger than the possible maximum number of "
                          f"paths. It has been set to k={self._k}.")
        kbest_check_limits(self._num_streams, self._k, self._num_symbols)
        self._list2llr = None
        if self._output == "bit":
            if not self._hard_out:
                self.list2llr = List2LLRSimple(self._num_bits_per_symbol) if list2llr is None else list2llr
        else:
            assert self._hard_out is True, "Soft-symbols are not supported for this detector."
        self._points_dev = None

    @property
    def list2llr(self):
        """``List2LLRSimple`` used for soft outputs; its ``llr_clip_val`` is read at every call."""
        return self._list2llr

    @list2llr.setter
    def list2llr(self, value):
        assert isinstance(value, List2LLR)
        if not isinstance(value, List2LLRSimple):
            raise NotImplementedError("KBestDetector computes LLRs inside its kernel: only List2LLRSimple is provided")
        self._list2llr = value

    def build(self, *input_shapes):
        assert input_shapes[1][-2] >= input_shapes[1][-1], \
            "The number of receive antennas cannot be smaller than the number of streams"

    def _kernel_args(self, dev):
        """(device points, k, real_rep, output, hard_out, llr_clip) of the C-ABI call."""
        if self._points_dev is None or self._points_dev.device != dev:
            dt = torch.float32 if self._use_real_rep else torch.complex64
            self._points_dev = torch.as_tensor(self._constellation).to(device=dev, dtype=dt).contiguous()
        clip = float(self._list2llr.llr_clip_val) if self._list2llr is not None else float("inf")
        return (self._points_dev, self._k, int(self._use_real_rep), int(self._output == "symbol"), int(self._hard_out),
                clip)

    def call(self, y, h, s):
        dev = self.device
        k, m = self._num_tx_streams, self._num_bits_out
        y, h, s, batch, mm, num = _dense_inputs(y, h, s, k, dev)
        out = detector_out(self._output, self._hard_out, m, batch + [k], dev)
        pts, kk, real_rep, symbol, hard, clip = self._kernel_args(dev)
        ws = detector_workspace(lib().sb_kbest_workspace_bytes(num, k, real_rep), dev)
        check(lib().sb_mimo_kbest(ptr(y), ptr(h), ptr(s), ptr(pts), ptr(out), ptr(ws), ws.numel(), num, mm, k, 2 ** m,
                                  kk, real_rep, symbol, hard, clip, current_stream()), "sb_mimo_kbest")
        return out


IT_MAX_STREAMS = 16
EP_MAX_POINTS = 256
PIC_MAX_POINTS = 1024


def iterative_check_limits(name, num_streams, num_points, max_points):
    """ValueError unless 1 <= num_streams <= 16 and num_points <= max_points (the limits of ``sb_mimo_ep`` /
    ``sb_mimo_mmse_pic`` and their OFDM variants: 256 points for EP, 1024 for MMSE-PIC)."""
    if not 1 <= int(num_streams) <= IT_MAX_STREAMS:
        raise ValueError(f"{name}: {num_streams} streams, supported are 1 ... {IT_MAX_STREAMS}")
    if num_points > max_points:
        raise ValueError(f"{name}: a {num_points}-point constellation, supported are at most {max_points} points")


def symbol_logits_to_llrs(logits, num_bits_per_symbol, method):
    """SymbolLogits2LLRs (mapping.py:927-967): ``[..., 2**m]`` point logits -> ``[..., m]`` LLRs, logsumexp (``"app"``)
    or max (``"maxlog"``) over the points whose label bit i (MSB first) is 1, minus the same over bit i = 0."""
    m = num_bits_per_symbol
    lab = ((torch.arange(2 ** m, device=logits.device)[:, None] >> torch.arange(m - 1, -1, -1, device=logits.device))
           & 1).bool()
    x = logits[..., :, None]
    ninf = torch.tensor(-float("inf"), dtype=logits.dtype, device=logits.device)
    red = (lambda v: torch.logsumexp(v, dim=-2)) if method == "app" else (lambda v: torch.amax(v, dim=-2))
    return red(torch.where(lab, x, ninf)) - red(torch.where(~lab, x, ninf))


class EPDetector(Block):
    """EPDetector(output, num_bits_per_symbol, hard_out=False, l=10, beta=0.9, precision=None)

    MIMO expectation-propagation detection (detection.py:1039-1312) on the fused ``sb_mimo_ep`` kernel: whitening with
    S, the real-valued equivalent channel, ``l`` EP iterations with damping ``beta`` over the PAM levels of the QAM
    (scaled to energy 1/2). ``call(y [..., M], h [..., M, K], s [..., M, M])`` -> LLRs / hard bits ``[..., K, m]``
    (``output="bit"``: maxlog per PAM, real part on the even bit positions) or QAM logits ``[..., K, 2**m]`` / int32
    indices ``[..., K]`` (``output="symbol"``, PAM2QAM). QAM only; limits: K <= 16 streams, at most 256 points
    (ValueError otherwise). M < K is accepted."""

    def __init__(self, output, num_bits_per_symbol, hard_out=False, l=10, beta=0.9, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        # same argument checks and error types as the reference (detection.py:1134-1153)
        assert output in ("bit", "symbol"), "Unknown output"
        assert l >= 1, "l must be a positive integer"
        assert 0.0 <= beta <= 1.0, "beta must be in [0,1]"
        m = int(num_bits_per_symbol)
        assert m >= 2 and m % 2 == 0, "EPDetector needs a QAM constellation (an even number of bits per symbol)"
        if 2 ** m > EP_MAX_POINTS:
            raise ValueError(f"EPDetector: {2 ** m}-QAM, supported are at most {EP_MAX_POINTS} points")
        self._output = output
        self._hard_out = bool(hard_out)
        self._l = int(l)
        self._beta = float(beta)
        self._num_bits_per_symbol = m
        self._levels = (np.real(pam(m // 2, precision="single")) / np.sqrt(2.0)).astype(np.float32)
        self._levels_dev = None

    def _kernel_args(self, dev):
        """(device PAM levels, num_points, l, beta, output, hard_out) of the C-ABI call."""
        if self._levels_dev is None or self._levels_dev.device != dev:
            self._levels_dev = torch.as_tensor(self._levels).to(dev).contiguous()
        return (self._levels_dev, 2 ** self._num_bits_per_symbol, self._l, self._beta, int(self._output == "symbol"),
                int(self._hard_out))

    def call(self, y, h, s):
        dev = self.device
        k = torch.as_tensor(h).shape[-1]
        iterative_check_limits("EPDetector", k, 2 ** self._num_bits_per_symbol, EP_MAX_POINTS)
        y, h, s, batch, mm, num = _dense_inputs(y, h, s, k, dev)
        out = detector_out(self._output, self._hard_out, self._num_bits_per_symbol, batch + [k], dev)
        lev, npts, l, beta, symbol, hard = self._kernel_args(dev)
        check(lib().sb_mimo_ep(ptr(y), ptr(h), ptr(s), ptr(lev), ptr(out), num, mm, k, npts, l, beta, symbol, hard,
                               current_stream()), "sb_mimo_ep")
        return out


class MMSEPICDetector(Block):
    """MMSEPICDetector(output, demapping_method="maxlog", num_iter=1, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    MIMO MMSE detection with parallel interference cancellation (detection.py:1314-1643) on the fused
    ``sb_mimo_mmse_pic`` kernel: whitening with S, then ``num_iter`` self-iterations of soft symbols from the a-priori
    LLRs, the unbiased PIC-MMSE estimate of every stream and demapping with the prior (``"app"`` or ``"maxlog"``); the
    output is the extrinsic information ``llr_d - llr_a``. ``call(y [..., M], h [..., M, K], s [..., M, M], prior)``:
    ``output="bit"``: prior = bit LLRs ``[..., K, m]`` -> LLRs / hard bits ``[..., K, m]``; ``output="symbol"``: prior =
    point logits ``[..., K, |C|]`` (converted to LLRs with the demapping method) -> logits ``[..., K, |C|]``
    (LLRs2SymbolLogits of the extrinsic LLRs) or their int32 argmax ``[..., K]``. Limits: K <= 16 streams, at most 1024
    points (ValueError otherwise). M < K is accepted."""

    def __init__(self, output, demapping_method="maxlog", num_iter=1, constellation_type=None, num_bits_per_symbol=None,
                 constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        # same argument checks and error types as the reference (detection.py:1456-1458)
        assert isinstance(num_iter, int), "num_iter must be an integer"
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        if num_iter < 1:
            raise ValueError(f"MMSEPICDetector: num_iter = {num_iter}, at least one self-iteration is needed")
        self._output = output
        self._method = demapping_method
        self._num_iter = num_iter
        self._hard_out = bool(hard_out)
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        if self._constellation.num_points > PIC_MAX_POINTS:
            raise ValueError(f"MMSEPICDetector: a {self._constellation.num_points}-point constellation, supported are "
                             f"at most {PIC_MAX_POINTS} points")

    @property
    def constellation(self):
        return self._constellation

    def _prior_llrs(self, prior, shape, dev):
        """Bit LLRs [*shape, m] (float32, contiguous) of a prior given in the output's kind."""
        m = self._constellation.num_bits_per_symbol
        pr = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
        if self._output == "symbol":
            pr = symbol_logits_to_llrs(pr, m, self._method)
        return pr.expand(shape + [m]).contiguous()

    def _finish(self, llr):
        """The kernel's extrinsic LLRs [..., m] (or hard bits) in the output's kind."""
        if self._output == "bit":
            return llr
        logits = llrs_to_symbol_logits(llr, self._constellation.num_bits_per_symbol)
        return torch.argmax(logits, dim=-1).to(torch.int32) if self._hard_out else logits

    def _kernel_args(self, dev):
        """(device points, num_points, num_iter, method, hard_out) of the C-ABI call."""
        pts = self._constellation().to(device=dev, dtype=torch.complex64).contiguous()
        return (pts, self._constellation.num_points, self._num_iter, 0 if self._method == "app" else 1,
                int(self._hard_out and self._output == "bit"))

    def call(self, y, h, s, prior):
        dev = self.device
        k, m = torch.as_tensor(h).shape[-1], self._constellation.num_bits_per_symbol
        iterative_check_limits("MMSEPICDetector", k, self._constellation.num_points, PIC_MAX_POINTS)
        y, h, s, batch, mm, num = _dense_inputs(y, h, s, k, dev)
        pr = self._prior_llrs(prior, batch + [k], dev)
        out = torch.empty(batch + [k, m], dtype=torch.float32, device=dev)
        pts, npts, num_iter, method, hard = self._kernel_args(dev)
        check(lib().sb_mimo_mmse_pic(ptr(y), ptr(h), ptr(s), ptr(pr), ptr(pts), ptr(out), num, mm, k, npts, num_iter,
                                     method, hard, current_stream()), "sb_mimo_mmse_pic")
        return self._finish(out)
