"""Generic linear encoder (mirror of fec/linear/encoding.py:10-140) on ``sb_gf2_encode`` (``csrc/linear_codes.cu``)."""
import numpy as np
import torch

from ...block import Block
from ...._lib import lib, check, ptr, current_stream
from ..utils import pcm2gm

_DTYPE_CODES = {torch.float32: 0, torch.float64: 1, torch.int32: 2, torch.int64: 3}


def _pack_rows(mat):
    """Bit-packed rows of a binary [k, n] matrix: ceil(n / 32) uint32 words per row, bit b of word w = column
    32 w + b."""
    k, n = mat.shape
    wn = (n + 31) // 32
    bits = np.zeros((k, wn * 32), np.uint8)
    bits[:, :n] = mat
    return np.packbits(bits.reshape(k, wn, 4, 8), axis=-1, bitorder="little").reshape(k, wn * 4).view(np.uint32)


def _check_binary_2d(enc_mat):
    enc_mat = np.asarray(enc_mat)
    if not ((enc_mat == 0) | (enc_mat == 1)).all():
        raise ValueError("enc_mat is not binary.")
    if enc_mat.ndim != 2:
        raise ValueError("enc_mat must be 2-D array.")
    return enc_mat


class LinearEncoder(Block):
    """LinearEncoder(enc_mat, *, is_pcm=False, precision=None)

    Encodes ``[..., k]`` information bits into ``[..., n]`` codewords c = u G mod 2 of the binary linear code with
    generator ``enc_mat`` [k, n] or, with ``is_pcm=True``, parity-check matrix ``enc_mat`` [n - k, n] (converted with
    :func:`~sionna_b200.phy.fec.utils.pcm2gm`, which needs a full-rank matrix). An input element contributes its lowest
    integer bit. As in the reference, floating inputs are first cast to the block's precision, so floating outputs
    are float32 (or float64 with ``precision="double"``, computed exactly); int32 / int64 inputs give outputs of the
    same type. Any ``k <= n`` whose bit-packed generator fits on the device; one kernel launch per call.

    Deviation: a non-binary or non-2-D ``enc_mat`` raises ``ValueError``, ``k > n`` ``AttributeError`` (as the
    reference) and a wrong last input dimension ``ValueError``."""

    _native_double = True

    def __init__(self, enc_mat, *, is_pcm=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if not isinstance(is_pcm, bool):
            raise TypeError("is_parity_check must be bool.")
        enc_mat = _check_binary_2d(enc_mat)
        gm = pcm2gm(enc_mat, verify_results=True) if is_pcm else enc_mat
        gm = np.asarray(gm).astype(np.uint8)
        self._k, self._n = int(gm.shape[0]), int(gm.shape[1])
        if not self._k <= self._n:
            raise AttributeError("Invalid matrix dimensions.")
        self._gm_np = gm
        self._gm = torch.from_numpy(gm).to(device=self.device, dtype=self.rdtype)
        self._coderate = self._k / self._n
        self._rows = torch.from_numpy(_pack_rows(gm).view(np.int32)).to(self.device)

    @property
    def k(self):
        """Number of information bits per codeword"""
        return self._k

    @property
    def n(self):
        """Codeword length"""
        return self._n

    @property
    def gm(self):
        """Generator matrix used for encoding"""
        return self._gm

    @property
    def coderate(self):
        """Coderate of the code"""
        return self._coderate

    def build(self, input_shape):
        if input_shape[-1] != self._k:
            raise ValueError(f"Last dimension must be of size k={self._k}.")

    def call(self, bits, /):
        if bits.shape[-1] != self._k:
            raise ValueError(f"Last dimension must be of size k={self._k}.")
        if bits.dtype not in _DTYPE_CODES:
            raise TypeError(f"Unsupported input dtype {bits.dtype}.")
        dev = self.device
        if self._rows.device != dev:
            self._rows = self._rows.to(dev)
        u = bits.to(dev).contiguous()
        batch = u.numel() // self._k
        c = torch.empty(list(u.shape[:-1]) + [self._n], dtype=u.dtype, device=dev)
        check(lib().sb_gf2_encode(ptr(u), ptr(c), _DTYPE_CODES[u.dtype], batch, self._k, self._n, ptr(self._rows),
                                  current_stream()), "sb_gf2_encode")
        return c
