"""Ordered statistics decoding (mirror of fec/linear/decoding.py:14-478) on ``sb_osd_decode``
(``csrc/linear_codes.cu``, DESIGN §3.13)."""
import ctypes as C
import itertools

import numpy as np
import scipy as sp
import torch

from ...block import Block
from ...._lib import lib, check, ptr, current_stream
from ..utils import pcm2gm, make_systematic


class _OSDCode:
    """Owns an ``sb_osd_code`` handle: the host-validated, bit-packed full-rank generator."""

    def __init__(self, gm):
        gm = np.ascontiguousarray(gm, np.uint8)
        h = C.c_void_p()
        check(lib().sb_osd_code_create(C.byref(h), ptr(gm), gm.shape[0], gm.shape[1]), "sb_osd_code_create")
        self.handle = h

    def __del__(self):
        if getattr(self, "handle", None):
            lib().sb_osd_code_destroy(self.handle)
            self.handle = None


class OSDecoder(Block):
    """OSDecoder(enc_mat=None, t=0, is_pcm=False, encoder=None, precision=None)

    Ordered statistics decoding of order ``t`` [Fossorier] for a binary linear code given by its generator ``enc_mat``
    [k, n], its parity-check matrix (``is_pcm=True``) or an ``encoder`` block, whose ``gm`` is then ``encoder(eye(k))``
    computed on the device (``LinearEncoder``, ``LDPC5GEncoder``, ``ConvEncoder``, ``TurboEncoder``, ...). Input
    ``[..., n]`` logits log p(1) / p(0) of any float dtype; output ``[..., n]`` hard decisions of the decoded codeword
    in the block's dtype. The steps are the reference's: clip to +-100, sort by |llr|, bring the generator to systematic
    form on the most reliable basis (MRB), re-encode the hard decisions of the k MRB positions and test every error
    pattern of weight 1 ... t there, one ``sb_osd_decode`` launch per call. ``t >= k`` is exact ML decoding.

    Deviations from the reference (DESIGN §1):

    - Candidates are ranked by the discrepancy D = sum of |llr| over the positions where they differ from the hard
      decisions. This orders them exactly as the reference's sum of log(1 + exp(llr (1 - 2 c))) does, but stays finite:
      the reference evaluates that sum in float32, which is inf as soon as a candidate contradicts an |llr| > 88.7, and
      then keeps the order-0 word.
    - The sort is stable (equal |llr| keep the lower index first); the reference's is not.
    - Among candidates with equal D the first in (order, combination rank over the MRB positions in reliability order)
      is kept; the output depends on nothing but the codeword's LLRs.
    - ``t > k`` acts as ``t = k``; n is limited to 1024 (``ValueError`` beyond).
    - ``precision="double"`` runs the float32 kernel (``PrecisionWarning``) and returns float64."""

    def __init__(self, enc_mat=None, t=0, is_pcm=False, encoder=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if not isinstance(is_pcm, bool):
            raise TypeError("is_pcm must be bool.")
        self._llr_max = 100.
        if enc_mat is not None:
            if isinstance(enc_mat, np.ndarray):
                if not np.array_equal(enc_mat, enc_mat.astype(bool)):
                    raise TypeError("PC matrix must be binary.")
            elif isinstance(enc_mat, (sp.sparse.csr_matrix, sp.sparse.csc_matrix)):
                if not np.array_equal(enc_mat.data, enc_mat.data.astype(bool)):
                    raise TypeError("PC matrix must be binary.")
                enc_mat = enc_mat.toarray()
            else:
                raise TypeError("Unsupported dtype of pcm.")
        if int(t) != t:
            raise TypeError("t must be int.")
        self._t = int(t)
        if self._t < 0:
            raise ValueError("t must be non-negative.")
        if encoder is not None:
            if encoder.k is None:
                raise AttributeError("It seems as if the encoder is not initialized or has no attribute k.")
            u = torch.eye(encoder.k, dtype=torch.float32, device=self.device).unsqueeze(0)
            gm = encoder(u).squeeze(0)
            gm_np = np.rint(gm.detach().to("cpu", torch.float64).numpy()).astype(np.int64)
            make_systematic(gm_np)                                      # full rank, ValueError otherwise
        else:
            if enc_mat is None:
                raise AttributeError("enc_mat cannot be None if no encoder is provided.")
            if is_pcm:
                gm_np = pcm2gm(enc_mat)
            else:
                make_systematic(enc_mat)
                gm_np = enc_mat
            gm_np = np.asarray(gm_np).astype(np.int64)
        self._gm = torch.from_numpy(gm_np).to(device=self.device, dtype=self.rdtype)
        self._k, self._n = int(gm_np.shape[0]), int(gm_np.shape[1])
        num_symbols = self._num_error_patterns(self._n, self._t) * self._n
        if num_symbols > 1e9:
            print(f"Note: Required memory complexity is large for the given code parameters and t={t}. Please "
                  "consider small batch-sizes to keep the inference complexity small and activate XLA mode if "
                  "possible.")
        if num_symbols > 1e11:
            raise ResourceWarning("Due to its high complexity, OSD is not feasible for the selected parameters. "
                                  "Please consider using a smaller value for t.")
        self._code = _OSDCode(gm_np)

    @property
    def gm(self):
        """Generator matrix of the code"""
        return self._gm

    @property
    def n(self):
        """Codeword length"""
        return self._n

    @property
    def k(self):
        """Number of information bits per codeword"""
        return self._k

    @property
    def t(self):
        """Order of the OSD algorithm"""
        return self._t

    def _num_error_patterns(self, n, t):
        """C(n, t), the number of error patterns of weight t in n positions."""
        return sp.special.comb(n, t, exact=True, repetition=False)

    def _gen_error_patterns(self, n, t):
        """All C(n, t) error patterns of weight t in n positions as [C(n, t), t] indices, itertools.combinations
        order (the kernel enumerates the same order without materialising it)."""
        return torch.tensor(list(itertools.combinations(range(n), t)), dtype=torch.int32).reshape(-1, t)

    def build(self, input_shape):
        if input_shape[-1] != self._n:
            raise ValueError(f" Last dimension must be of size n={self._n}.")

    def call(self, llr_ch, /):
        if llr_ch.shape[-1] != self._n:
            raise ValueError(f" Last dimension must be of size n={self._n}.")
        x = llr_ch.to(device=self.device, dtype=torch.float32).contiguous()
        batch = x.numel() // self._n
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
        check(lib().sb_osd_decode(self._code.handle, ptr(x), ptr(out), batch, self._t, current_stream()),
              "sb_osd_decode")
        return out
