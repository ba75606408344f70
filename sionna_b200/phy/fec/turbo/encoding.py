"""Turbo encoder (mirror of fec/turbo/encoding.py:16-421) composed of existing kernels: ``sb_gather_rows`` interleaves,
``sb_conv_encode`` runs both RSC component encoders, ``sb_gather_rows`` multiplexes, terminates and punctures."""
import math

import numpy as np
import torch

from ...block import Block
from ...config import config
from ...._lib import lib, check, ptr, current_stream
from ..conv.utils import Trellis
from ..interleaving import RandomInterleaver, Turbo3GPPInterleaver
from .utils import polynomial_selector, puncture_pattern, TurboTermination


def interleaver_perm(interleaver, k):
    """int64 [k]: the permutation pi the turbo code's interleaver applies to k bits (u2[i] = u[pi(i)])."""
    if isinstance(interleaver, Turbo3GPPInterleaver):
        return interleaver.perm(k)
    return interleaver.perm(k)[0]


def turbo_layout(k, mu, rate, terminate):
    """Index tables of a turbo codeword of k information bits (encoding.py:391-421, decoding.py:254-355).

    The component codewords are held side by side as [2, 2 T] (T = k + mu if terminated): step t of encoder d at
    d 2 T + 2 t (systematic) and + 1 (parity). Returns (mux [n], demux [4 T], perm-independent part of demux):
    mux[j] is the component position turbo bit j comes from, -1 for the zero padding of the termination symbols;
    demux[d 2 T + 2 t + b] is the turbo bit that position reads, -1 if punctured or absent. Decoder 2's systematic
    positions (t < k) are left -1 here; the caller fills them through the interleaver."""
    T = k + (mu if terminate else 0)
    pre = []                                                  # pre-puncturing turbo stream, 3 bits per symbol
    for t in range(k):
        pre += [2 * t, 2 * t + 1, 2 * T + 2 * t + 1]         # x1(t), z1(t), z2(t)
    if terminate:
        term = TurboTermination(mu + 1, conv_n=2)
        tb = [2 * t + b for t in range(k, T) for b in range(2)] + [2 * T + 2 * t + b for t in range(k, T) for b in range(2)]
        tb = np.array(tb) + 1                                 # shifted by one so that the zero padding becomes -1
        pre += list(term.termbits_conv2turbo(tb[:2 * mu], tb[2 * mu:]) - 1)
    pattern = puncture_pattern(rate, 1 / 2)
    keep = np.tile(pattern, (math.ceil(len(pre) / 3 / len(pattern)), 1))[:len(pre) // 3].reshape(-1)
    pre = np.array(pre, np.int64)
    mux = pre[keep]
    rank = np.full(len(pre), -1, np.int64)
    rank[keep] = np.arange(int(keep.sum()))
    demux = np.full(4 * T, -1, np.int64)
    for t in range(k):
        demux[2 * t:2 * t + 2] = rank[3 * t:3 * t + 2]
        demux[2 * T + 2 * t + 1] = rank[3 * t + 2]
    if terminate:
        base = 3 * k
        for s in range(mu):
            demux[2 * (k + s):2 * (k + s) + 2] = rank[base + 2 * s:base + 2 * s + 2]
            demux[2 * T + 2 * (k + s):2 * T + 2 * (k + s) + 2] = rank[base + 2 * mu + 2 * s:base + 2 * mu + 2 * s + 2]
    return mux, demux, rank


def dev_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(config.device)


def gather(x, idx_dev, rows, cols_out, cols_in):
    """out [batch, rows, cols_out] = x [batch, cols_in] through the index rows idx_dev [rows, cols_out] (-1: 0)."""
    batch = x.numel() // cols_in
    out = torch.empty((batch, rows, cols_out), dtype=torch.float32, device=x.device)
    check(lib().sb_gather_rows(ptr(x), ptr(idx_dev), ptr(out), batch, rows, cols_out, 1, cols_in, 1, current_stream()),
          "sb_gather_rows")
    return out


class TurboEncoder(Block):
    """TurboEncoder(gen_poly=None, constraint_length=3, rate=1/3, terminate=False, interleaver_type='3GPP',
    precision=None)

    Encodes bits ``[..., k]`` into a turbo codeword ``[..., n]`` (encoding.py:16-421): two rate-1/2 RSC encoders, the
    second fed through the interleaver (``Turbo3GPPInterleaver`` or a ``RandomInterleaver`` with a fixed seed), output
    symbols (x1, z1, z2), then the termination symbols, punctured to rate 1/2 if asked. ``gen_poly``: two equally long
    0/1 strings, the feedback polynomial first; otherwise ``constraint_length`` 3 ... 6 selects turbo's tabulated code.
    With ``terminate`` n = (k + ceil(4 mu / 3)) / rate."""

    def __init__(self, gen_poly=None, constraint_length=3, rate=1 / 3, terminate=False, interleaver_type="3GPP",
                 precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if gen_poly is not None:
            if not all(isinstance(p, str) for p in gen_poly):
                raise TypeError("Each element of gen_poly must be a string.")
            if not all(len(p) == len(gen_poly[0]) for p in gen_poly):
                raise ValueError("Each polynomial must be of same length.")
            if not all(all(c in "01" for c in p) for p in gen_poly):
                raise ValueError("Each Polynomial must be a string of 0/1 s.")
            if len(gen_poly) != 2:
                raise ValueError("Generator polynomials need to be of rate-1/2")
            self._gen_poly = gen_poly
        else:
            if constraint_length not in (3, 4, 5, 6):
                raise ValueError("Constraint length must be between 3 and 6.")
            self._gen_poly = polynomial_selector(constraint_length)
        if rate not in (1 / 2, 1 / 3):
            raise ValueError("Invalid coderate.")
        if not isinstance(terminate, bool):
            raise TypeError("terminate must be bool.")
        if interleaver_type not in ("3GPP", "random"):
            raise ValueError("Invalid interleaver_type.")
        self._coderate_desired = rate
        self._coderate = rate
        self._terminate = terminate
        self._interleaver_type = interleaver_type
        self._coderate_conv = 1 / len(self._gen_poly)
        self._punct_pattern = puncture_pattern(rate, self._coderate_conv)
        self._trellis = Trellis(self._gen_poly, rsc=True)
        self._mu = self._trellis._mu
        self._conv_k = self._trellis.conv_k
        self._conv_n = self._trellis.conv_n
        self._ns = self._trellis.ns
        self._k = None
        self._n = None
        if terminate:
            self.turbo_term = TurboTermination(self._mu + 1, conv_n=self._conv_n)
        if interleaver_type == "3GPP":
            self.internal_interleaver = Turbo3GPPInterleaver()
        else:
            self.internal_interleaver = RandomInterleaver(keep_batch_constant=True, keep_state=True, axis=-1)
        self._polys = np.array([int(p, 2) for p in self._gen_poly], np.int32)
        self._tables = None

    @property
    def gen_poly(self):
        """Generator polynomials of the component code"""
        return self._gen_poly

    @property
    def constraint_length(self):
        """Constraint length of the component encoders"""
        return self._mu + 1

    @property
    def coderate(self):
        """Rate of the code; with termination the true rate once k is known"""
        if self.terminate and self._k is None:
            print("Note that, due to termination, the true coderate is lower than the returned design rate. The exact "
                  "true rate is dependent on the value of k and hence cannot be computed before the first call().")
        elif self.terminate and self._k is not None:
            term_factor = 1 + math.ceil(4 * self._mu / 3) / self._k
            self._coderate = self._coderate_desired / term_factor
        return self._coderate

    @property
    def trellis(self):
        """Trellis of the component code"""
        return self._trellis

    @property
    def terminate(self):
        """Whether the component encoders are terminated"""
        return self._terminate

    @property
    def punct_pattern(self):
        """Puncturing pattern (bool [period, 3]) of the turbo codeword"""
        return self._punct_pattern

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
        self._k = int(input_shape[-1])
        if self._interleaver_type == "3GPP" and self._k > 6144:
            raise ValueError("3GPP Turbo Codes define Interleavers only upto frame lengths of 6144")
        self.num_syms = self._k // self._conv_k
        mux, _, _ = turbo_layout(self._k, self._mu, self._coderate_desired, self._terminate)
        self._n = len(mux)
        perm = interleaver_perm(self.internal_interleaver, self._k)
        self._tables = (dev_i32(np.stack([np.arange(self._k), perm])), dev_i32(mux))

    def call(self, bits, /):
        if bits.shape[-1] != self._k or self._tables is None:
            self.build(bits.shape)
        k, T = self._k, self._k + (self._mu if self._terminate else 0)
        u = bits.to(device=self.device, dtype=torch.float32).reshape(-1, k).contiguous()
        batch = u.shape[0]
        u2 = gather(u, self._tables[0], 2, k, k)                                  # [batch, 2, k]: u, pi(u)
        x2 = torch.empty((batch, 2, 2 * T), dtype=torch.float32, device=u.device)
        if batch:
            check(lib().sb_conv_encode(ptr(u2), ptr(x2), 2 * batch, k, ptr(self._polys), self._conv_n, self._mu + 1, 1,
                                       int(self._terminate), current_stream()), "sb_conv_encode")
        x = gather(x2, self._tables[1], 1, self._n, 4 * T)
        return x.to(self.rdtype).reshape(*bits.shape[:-1], self._n)
