"""Turbo decoder (mirror of fec/turbo/decoding.py:15-435) on ``sb_turbo_decode`` (``csrc/conv.cu``, DESIGN §3.12): one
``sb_gather_rows`` depunctures and splits the codeword into the two component codewords, one launch runs every
iteration of both BCJR component decoders."""

import numpy as np
import torch

from ...block import Block
from ...._lib import Handle, lib, check, ptr, current_stream
from ..conv.utils import Trellis, _trellis_tables
from ..interleaving import RandomInterleaver, Turbo3GPPInterleaver
from .encoding import interleaver_perm, turbo_layout, dev_i32, gather
from .utils import polynomial_selector, puncture_pattern, TurboTermination


class TurboDecoder(Block):
    """TurboDecoder(encoder=None, gen_poly=None, rate=1/3, constraint_length=None, interleaver='3GPP', terminate=False,
    num_iter=6, hard_out=True, algorithm='map', precision=None)

    Iterative decoding of turbo codewords ``[..., n]`` of logits (decoding.py:15-435): ``num_iter`` iterations of two
    BCJR component decoders exchanging extrinsic LLRs clipped to +-20. Returns ``[..., k]`` estimates of the information
    bits: decoder 2's APP LLRs deinterleaved, or ``llr > 0`` with ``hard_out``. With ``encoder`` the code, termination
    and interleaver (the same instance, so a random interleaver's seed matches) come from it. ``algorithm``: "map" and
    "log" (both the exact function, evaluated in the log domain) or "maxlog".

    Deviations: the rate taken from ``encoder`` is its design rate (the reference reads its current ``_coderate``, which
    is the terminated true rate once ``encoder.coderate`` has been read and then fails); the decoder does not print the
    input dtype on every call. ``precision="double"`` takes and returns float64 and runs the fp32 kernel
    (``PrecisionWarning``)."""

    def __init__(self, encoder=None, gen_poly=None, rate=1 / 3, constraint_length=None, interleaver="3GPP",
                 terminate=False, num_iter=6, hard_out=True, algorithm="map", precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if encoder is not None:
            self._coderate = encoder._coderate_desired
            self._gen_poly = encoder._gen_poly
            self._terminate = encoder.terminate
            self._trellis = encoder.trellis
            assert self._trellis.rsc is True
            self.rsc = True
            self.internal_interleaver = encoder.internal_interleaver
        else:
            if gen_poly is not None:
                if not all(isinstance(p, str) for p in gen_poly):
                    raise TypeError("Each polynomial must be a string.")
                if not all(len(p) == len(gen_poly[0]) for p in gen_poly):
                    raise ValueError("Each polynomial must be of same length.")
                if not all(all(c in "01" for c in p) for p in gen_poly):
                    raise ValueError("Each polynomial must be a string of 0's and 1's.")
                self._gen_poly = gen_poly
            else:
                if constraint_length not in (3, 4, 5, 6):
                    raise ValueError("Constraint length must be between 3 and 6.")
                self._gen_poly = polynomial_selector(constraint_length)
            if rate not in (1 / 2, 1 / 3):
                raise ValueError("rate must be 1/3 or 1/2.")
            self._coderate = rate
            if not isinstance(terminate, bool):
                raise TypeError("terminate must be bool.")
            self._terminate = terminate
            if interleaver not in ("3GPP", "random"):
                raise ValueError("interleaver must be 3GPP or random.")
            if interleaver == "3GPP":
                self.internal_interleaver = Turbo3GPPInterleaver(precision=precision)
            else:
                self.internal_interleaver = RandomInterleaver(keep_batch_constant=True, keep_state=True, axis=-1,
                                                              precision=precision)
            self.rsc = True
            self._trellis = Trellis(self._gen_poly, rsc=True)
        if not isinstance(hard_out, bool):
            raise TypeError("hard_out must be bool.")
        if algorithm not in ("map", "log", "maxlog"):
            raise ValueError("algorithm must be one of map, log or maxlog")
        self._conv_k = self._trellis.conv_k
        self._mu = self._trellis._mu
        self._conv_n = self._trellis.conv_n
        self._ns = self._trellis.ns
        if self._conv_k != 1 or self._conv_n != 2:
            raise NotImplementedError("Only single bit stream support.")
        self._coderate_conv = 1 / len(self._gen_poly)
        self.punct_pattern = puncture_pattern(self._coderate, self._coderate_conv)
        self._k = None
        self._n = None
        if self._terminate:
            self.turbo_term = TurboTermination(self._mu + 1, conv_n=self._conv_n)
            self._num_term_bits = 3 * self.turbo_term.get_num_term_syms()
        else:
            self._num_term_bits = 0
        self.num_iter = num_iter
        self._hard_out = hard_out
        self._algorithm = algorithm
        self._tables = _trellis_tables(self._trellis)
        self._demux = None
        self._perm = None

    @property
    def gen_poly(self):
        """Generator polynomials of the component code"""
        return self._gen_poly

    @property
    def constraint_length(self):
        """Constraint length of the component code"""
        return self._mu + 1

    @property
    def coderate(self):
        """Design rate of the code"""
        return self._coderate

    @property
    def trellis(self):
        """Trellis of the component code"""
        return self._trellis

    @property
    def k(self):
        """Number of information bits per codeword"""
        if self._k is None:
            print("Note: The value of k cannot be computed before the first call().")
        return self._k

    @property
    def n(self):
        """Number of codeword bits"""
        if self._n is None:
            print("Note: The value of n cannot be computed before the first call().")
        return self._n

    def build(self, input_shape):
        n = int(input_shape[-1])
        if self.coderate == 1 / 2 and n % 2 != 0:
            raise ValueError("Codeword length should be a multiple of 2")
        turbo_n_preterm = int(n * self.coderate * 3) - self._num_term_bits
        if turbo_n_preterm % 3 != 0 or turbo_n_preterm < 3:
            raise ValueError("Invalid codeword length for a terminated Turbo code")
        self._n = n
        self._k = turbo_n_preterm // 3
        self._convenc_numsyms = self._k + (self._mu if self._terminate else 0)
        self._demux = None

    def _prepare(self):
        """Device demultiplexing table and interleaver handle of the current k."""
        k, T = self._k, self._convenc_numsyms
        _, demux, rank = turbo_layout(k, self._mu, self._coderate, self._terminate)
        perm = interleaver_perm(self.internal_interleaver, k)
        demux[2 * T + 2 * np.arange(k)] = rank[3 * perm]              # decoder 2's systematic LLRs, through pi
        self._demux = dev_i32(demux)
        perm = np.ascontiguousarray(perm, np.int32)
        self._perm = Handle("turbo_perm", ptr(perm), len(perm))   # checked by the library to be a permutation

    def call(self, llr_ch, /):
        if llr_ch.shape[-1] != self._n:
            self.build(llr_ch.shape)
        if self._demux is None:
            self._prepare()
        k, T = self._k, self._convenc_numsyms
        y = llr_ch.to(device=self.device, dtype=torch.float32).reshape(-1, self._n).contiguous()
        batch = y.shape[0]
        y2 = gather(y, self._demux.to(y.device), 1, 4 * T, self._n)  # [batch, 1, 2 * 2T]: both component codewords
        out = torch.empty((batch, k), dtype=torch.float32, device=y.device)
        nbytes = lib().sb_turbo_workspace_bytes(batch, k, int(self._terminate), self._ns)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device) if nbytes else None
        fr, op, ip = self._tables
        check(lib().sb_turbo_decode(ptr(y2), self._perm.handle, ptr(out), batch, k, int(self.num_iter),
                                    ("map", "log", "maxlog").index(self._algorithm), int(self._terminate),
                                    int(self._hard_out), ptr(fr), ptr(op), ptr(ip), self._ns, self._conv_n, ptr(ws),
                                    0 if ws is None else ws.numel(), current_stream()), "sb_turbo_decode")
        return out.to(self.rdtype).reshape(*llr_ch.shape[:-1], k)
