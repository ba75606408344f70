"""Convolutional encoder (mirror of fec/conv/encoding.py:11-292) on ``sb_conv_encode`` (``csrc/conv.cu``)."""
import numpy as np
import torch

from ...block import Block
from ...._lib import lib, check, ptr, current_stream
from .utils import Trellis, _select_gen_poly


class ConvEncoder(Block):
    """ConvEncoder(gen_poly=None, rate=1/2, constraint_length=3, rsc=False, terminate=False, precision=None)

    Encodes bits ``[..., k]`` into a rate-1/n convolutional codeword ``[..., n]``; the n bits of a step are adjacent.
    ``gen_poly``: tuple of equally long 0/1 strings (first character: coefficient of the newest bit); otherwise
    ``rate`` (1/2, 1/3) and ``constraint_length`` (3 ... 8) select a tabulated code. ``rsc``: recursive systematic
    code with the first polynomial as feedback. ``terminate``: K - 1 termination steps drive the register to zero
    (for RSC codes with the feedback bits as inputs), so n = (k + K - 1) / rate."""

    def __init__(self, gen_poly=None, rate=1 / 2, constraint_length=3, rsc=False, terminate=False, precision=None,
                 **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._gen_poly = _select_gen_poly(gen_poly, rate, constraint_length,
                                          "Each element of gen_poly must be a string.")
        self._rsc = rsc
        self._terminate = terminate
        self._coderate_desired = 1 / len(self._gen_poly)
        self._coderate = self._coderate_desired
        self._trellis = Trellis(self._gen_poly, rsc=rsc)
        self._mu = self._trellis._mu
        self._conv_k = self._trellis.conv_k
        self._conv_n = self._trellis.conv_n
        self._ni = 2 ** self._conv_k
        self._no = 2 ** self._conv_n
        self._ns = self._trellis.ns
        self._polys = np.array([int(p, 2) for p in self._gen_poly], np.int32)
        self._k = None
        self._n = None

    @property
    def gen_poly(self):
        """Generator polynomials used by the encoder"""
        return self._gen_poly

    @property
    def coderate(self):
        """Rate of the code; with termination the true rate k / n once k is known"""
        if self.terminate and self._k is None:
            print("Note that, due to termination, the true coderate is lower than the returned design rate. "
                  "The exact true rate is dependent on the value of k and hence cannot be computed before the first "
                  "call().")
        elif self.terminate and self._k is not None:
            self._coderate = self._coderate_desired * self._k / (self._k + self._mu)
        return self._coderate

    @property
    def trellis(self):
        """Trellis of the code"""
        return self._trellis

    @property
    def terminate(self):
        """Whether the codewords are terminated in the all-zero state"""
        return self._terminate

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
        self._n = (self._k + (self._mu if self._terminate else 0)) * self._conv_n
        self.num_syms = self._k

    def call(self, bits, /):
        if bits.shape[-1] != self._k:
            self.build(bits.shape)
        u = bits.to(device=self.device, dtype=torch.float32).reshape(-1, self._k).contiguous()
        x = torch.empty((u.shape[0], self._n), dtype=torch.float32, device=u.device)
        check(lib().sb_conv_encode(ptr(u), ptr(x), u.shape[0], self._k, ptr(self._polys), self._conv_n, self._mu + 1,
                                   int(self._rsc), int(self._terminate), current_stream()), "sb_conv_encode")
        return x.to(self.rdtype).reshape(*bits.shape[:-1], self._n)
