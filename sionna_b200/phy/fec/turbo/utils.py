"""Host utilities of turbo codes (mirror of fec/turbo/utils.py:10-295): the component-code selector, the puncturing
pattern and the termination-bit bookkeeping. Nothing here touches the device."""
import math

import numpy as np

from ...block import Object


def polynomial_selector(constraint_length):
    """Generator polynomials (feedback first) of the rate-1/2 RSC component code of the given constraint length 3 ... 6
    (utils.py:10-46). These are turbo's own table, not ``conv.polynomial_selector``'s."""
    if not isinstance(constraint_length, int):
        raise TypeError("constraint_length must be int.")
    if not 2 < constraint_length < 7:
        raise ValueError("Unsupported constraint_length.")
    return {3: ("111", "101"), 4: ("1011", "1101"), 5: ("10011", "11011"), 6: ("111101", "101011")}[constraint_length]


def puncture_pattern(turbo_coderate, conv_coderate):
    """bool [period, 3]: which of (systematic, parity 1, parity 2) each turbo symbol keeps (utils.py:49-78); row r of the
    codeword uses row r mod period. Rates 1/3 and 1/2 over a rate-1/2 component code."""
    if conv_coderate != 1 / 2:
        raise ValueError("Only rate-1/2 component codes are supported.")
    if turbo_coderate == 1 / 2:
        pattern = [[1, 1, 0], [1, 0, 1]]
    elif turbo_coderate == 1 / 3:
        pattern = [[1, 1, 1]]
    else:
        raise NotImplementedError("turbo_coderate not supported")
    return np.array(pattern, bool)


class TurboTermination(Object):
    """TurboTermination(constraint_length, conv_n=2, num_conv_encs=2, num_bitstreams=3)

    Moves termination bits between the two component codewords and the turbo codeword (utils.py:81-295): the 2 mu
    termination bits of encoder 1 ([x1(K), z1(K), ..., x1(K+mu-1), z1(K+mu-1)]), then encoder 2's, then zeros up to a
    multiple of ``num_bitstreams``."""

    def __init__(self, constraint_length, conv_n=2, num_conv_encs=2, num_bitstreams=3, **kwargs):
        super().__init__(**kwargs)
        self.mu_ = int(constraint_length) - 1
        self.conv_n = int(conv_n)
        if int(num_conv_encs) != 2:
            raise NotImplementedError("Only num_conv_encs=2 supported.")
        self.num_conv_encs = int(num_conv_encs)
        self.num_bitstreams = int(num_bitstreams)

    def get_num_term_syms(self):
        """Number of turbo symbols (``num_bitstreams`` bits each) the termination bits occupy."""
        return math.ceil(self.conv_n * self.num_conv_encs * self.mu_ / self.num_bitstreams)

    def termbits_conv2turbo(self, term_bits1, term_bits2):
        """[..., 3 * num_term_syms]: both encoders' termination bits in order, then zero padding."""
        tb = np.concatenate([np.asarray(term_bits1), np.asarray(term_bits2)], axis=-1)
        extra = self.num_bitstreams * self.get_num_term_syms() - tb.shape[-1]
        if extra > 0:
            tb = np.concatenate([tb, np.zeros(tb.shape[:-1] + (extra,), tb.dtype)], axis=-1)
        return tb

    def term_bits_turbo2conv(self, term_bits):
        """The termination part of a turbo codeword split into encoder 1's and encoder 2's 2 mu values."""
        term_bits = np.asarray(term_bits)
        if term_bits.shape[-1] % self.num_bitstreams:
            raise ValueError("The termination part must hold whole turbo symbols.")
        m = self.conv_n * self.mu_
        return term_bits[..., :m], term_bits[..., m:2 * m]
