"""MIMO detection (mirror of /root/reference/src/sionna/phy/mimo/detection.py:24-537): linear and maximum-likelihood."""
import numpy as np
import torch

from ..._lib import lib, check, ptr, current_stream
from ..block import Block
from ..mapping import Constellation, Demapper
from .equalization import lmmse_equalizer


class LinearDetector(Block):
    """LinearDetector(equalizer, output, demapping_method, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    Equaliser followed by a demapper (detection.py:87-143): ``call(y, h, s)`` -> LLRs ``[..., K, num_bits_per_symbol]``
    (``output="bit"``). ``equalizer`` is ``"lmmse"`` or a callable ``(y, h, s) -> (x_hat, no_eff)``."""

    def __init__(self, equalizer, output, demapping_method, constellation_type=None, num_bits_per_symbol=None,
                 constellation=None, hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._output = output
        self._hard_out = hard_out
        # same argument checks and error types as the reference (detection.py:103-115)
        if isinstance(equalizer, str):
            assert equalizer in ["lmmse", "zf", "mf"], "Unknown equalizer."
            if equalizer != "lmmse":
                raise NotImplementedError(f"equalizer='{equalizer}': only the LMMSE equaliser has a kernel here "
                                          "(pass a callable (y, h, s) -> (x_hat, no_eff) for anything else).")
            equalizer = lmmse_equalizer
        self._equalizer = equalizer
        assert output in ("bit", "symbol"), "Unknown output"
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        if output != "bit":
            raise NotImplementedError("output='symbol' (SymbolDemapper) is not provided; use output='bit'.")
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        self._demapper = Demapper(demapping_method, constellation=self._constellation, hard_out=hard_out,
                                  precision=precision)

    def call(self, y, h, s):
        x_hat, no_eff = self._equalizer(y, h, s)
        z = self._demapper(x_hat, no_eff)
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


def ml_workspace(num_problems, num_streams, device):
    """Workspace of ``sb_mimo_ml`` / ``sb_ofdm_ml`` from PyTorch's caching allocator (whitened triangular records and
    output positions, ``sb_ml_workspace_bytes``)."""
    n = int(lib().sb_ml_workspace_bytes(int(num_problems), int(num_streams)))
    return torch.empty(max(n, 8), dtype=torch.uint8, device=device)


def llrs_to_symbol_logits(llrs, num_bits_per_symbol):
    """LLRs2SymbolLogits (mapping.py:1045-1059): ``[..., m]`` bit LLRs -> ``[..., 2**m]`` point logits
    ``sum_i log_sigmoid(a_ci * llr_i)``, a_ci = +1 / -1 for label bit i (MSB first) of point c equal to 1 / 0."""
    m = num_bits_per_symbol
    a = 2.0 * ((torch.arange(2 ** m, device=llrs.device)[:, None] >> torch.arange(m - 1, -1, -1, device=llrs.device)) & 1) - 1.0
    return torch.nn.functional.logsigmoid(llrs[..., None, :] * a.to(llrs.dtype)).sum(-1)


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
        h = torch.as_tensor(h).to(device=dev, dtype=torch.complex64)
        mm = h.shape[-2]
        if h.shape[-1] != k:
            raise ValueError(f"h must have num_streams = {k} as last dimension")
        batch = torch.broadcast_shapes(tuple(torch.as_tensor(y).shape[:-1]), tuple(h.shape[:-2]),
                                       tuple(torch.as_tensor(s).shape[:-2]))
        y = torch.as_tensor(y).to(device=dev, dtype=torch.complex64).expand(list(batch) + [mm]).contiguous()
        h = h.expand(list(batch) + [mm, k]).contiguous()
        s = torch.as_tensor(s).to(device=dev, dtype=torch.complex64).expand(list(batch) + [mm, mm]).contiguous()
        num = int(np.prod(batch)) if len(batch) else 1
        pr = None
        if prior is not None:
            pr = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if self._output == "bit":
                pr = llrs_to_symbol_logits(pr, m)
            pr = pr.expand(list(batch) + [k, npts]).contiguous()
        if self._output == "bit":
            out = torch.empty(list(batch) + [k, m], dtype=torch.float32, device=dev)
        elif self._hard_out:
            out = torch.empty(list(batch) + [k], dtype=torch.int32, device=dev)
        else:
            out = torch.empty(list(batch) + [k, npts], dtype=torch.float32, device=dev)
        pts = self._constellation().to(device=dev, dtype=torch.complex64).contiguous()
        ws = ml_workspace(num, k, dev)
        check(lib().sb_mimo_ml(ptr(y), ptr(h), ptr(s), ptr(pr), ptr(pts), ptr(out), ptr(ws), ws.numel(), num, mm, k, npts,
                               self._method, int(self._output == "symbol"), int(self._hard_out), current_stream()),
              "sb_mimo_ml")
        return out
