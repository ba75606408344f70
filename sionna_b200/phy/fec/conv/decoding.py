"""Viterbi and BCJR decoding of convolutional codes (mirror of fec/conv/decoding.py:19-943) on ``sb_viterbi_decode`` /
``sb_bcjr_decode`` (``csrc/conv.cu``, DESIGN §3.11)."""
import torch

from ...block import Block
from ...._lib import lib, check, ptr, current_stream
from .utils import Trellis, _select_gen_poly, _trellis_tables


class _TrellisDecoder(Block):
    """Code set-up and length bookkeeping shared by both decoders (decoding.py:94-213, 388-401, 533-661, 888-897)."""

    def __init__(self, encoder, gen_poly, rate, constraint_length, rsc, terminate, precision, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if encoder is not None:
            self._gen_poly = encoder.gen_poly
            self._trellis = encoder.trellis
            self._terminate = encoder.terminate
        else:
            self._gen_poly = _select_gen_poly(gen_poly, rate, constraint_length, "Each polynomial must be a string.")
            self._trellis = Trellis(self._gen_poly, rsc=rsc)
            self._terminate = terminate
        self._coderate_desired = 1 / len(self._gen_poly)
        self._coderate = self._coderate_desired
        self._mu = self._trellis._mu
        self._conv_k = self._trellis.conv_k
        self._conv_n = self._trellis.conv_n
        self._ni = 2 ** self._conv_k
        self._no = 2 ** self._conv_n
        self._ns = self._trellis.ns
        self._tables = _trellis_tables(self._trellis)
        self._k = None
        self._n = None
        self._num_syms = None

    @property
    def gen_poly(self):
        """Generator polynomials of the code"""
        return self._gen_poly

    @property
    def coderate(self):
        """Rate of the code; with termination the true rate once n is known"""
        if self.terminate and self._n is None:
            print("Note that, due to termination, the true coderate is lower than the returned design rate. "
                  "The exact true rate is dependent on the value of n and hence cannot be computed before the first "
                  "call().")
            self._coderate = self._coderate_desired
        elif self.terminate and self._n is not None:
            self._coderate = (self._coderate_desired * self._n - self._mu) / self._n
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

    def build(self, input_shape, **kwargs):
        n = int(input_shape[-1])
        if n % self._conv_n != 0:
            raise ValueError("Length of codeword should be divisible by number of output bits per symbol.")
        num_syms = n // self._conv_n
        k = num_syms - (self._mu if self._terminate else 0)
        if k < 1:
            raise ValueError(f"A terminated codeword needs more than {self._mu} symbols; n = {n} has {num_syms}.")
        self._n, self._num_syms, self._k = n, num_syms, k

    def _rows(self, x):
        if x.shape[-1] != self._n:
            self.build(x.shape)
        return x.to(device=self.device, dtype=torch.float32).reshape(-1, self._n).contiguous()

    def _workspace(self, fn, batch, dev):
        nbytes = fn(batch, self._num_syms, self._ns)
        return torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None


class ViterbiDecoder(_TrellisDecoder):
    """ViterbiDecoder(*, encoder=None, gen_poly=None, rate=1/2, constraint_length=3, rsc=False, terminate=False,
    method="soft_llr", return_info_bits=True, precision=None)

    Maximum-likelihood sequence decoding of logits ``[..., n]`` (decoding.py:19-453). ``method`` "soft_llr": branch
    metric sum_j llr_j (1 - 2 b_j); "hard": Manhattan distance of the rounded input bits. Returns the information
    bits ``[..., k]``, or the re-encoded survivor ``[..., n]`` with ``return_info_bits=False``. k = n / conv_n minus
    K - 1 termination steps if ``terminate``; it follows the input's last dimension on every call."""

    def __init__(self, *, encoder=None, gen_poly=None, rate=1 / 2, constraint_length=3, rsc=False, terminate=False,
                 method="soft_llr", return_info_bits=True, precision=None, **kwargs):
        super().__init__(encoder, gen_poly, rate, constraint_length, rsc, terminate, precision, **kwargs)
        if method not in ("soft_llr", "hard"):
            raise ValueError("method must be `soft_llr` or `hard`.")
        self._method = method
        self._return_info_bits = return_info_bits

    def call(self, inputs, /):
        y = self._rows(inputs)
        out_len = self._k if self._return_info_bits else self._n
        out = torch.empty((y.shape[0], out_len), dtype=torch.float32, device=y.device)
        ws = self._workspace(lib().sb_viterbi_workspace_bytes, y.shape[0], y.device)
        fr, op, ip = self._tables
        check(lib().sb_viterbi_decode(ptr(y), ptr(out), y.shape[0], self._num_syms, self._k,
                                      0 if self._method == "soft_llr" else 1, int(self._terminate),
                                      int(self._return_info_bits), ptr(fr), ptr(op), ptr(ip), self._ns, self._conv_n,
                                      ptr(ws), 0 if ws is None else ws.numel(), current_stream()),
              "sb_viterbi_decode")
        return out.to(self.rdtype).reshape(*inputs.shape[:-1], out_len)


class BCJRDecoder(_TrellisDecoder):
    """BCJRDecoder(encoder=None, gen_poly=None, rate=1/2, constraint_length=3, rsc=False, terminate=False,
    hard_out=True, algorithm="map", precision=None)

    Symbol-wise MAP decoding (decoding.py:456-943): ``dec(llr_ch, llr_a=None)`` with channel logits ``[..., n]`` and
    optional a-priori logits ``[..., n / conv_n]`` of the input bits (termination steps included). Returns the APP
    logits of the k information bits, or ``llr > 0`` with ``hard_out``. ``algorithm``: "map" (exact; evaluated in the
    log domain, which is the same function and cannot overflow), "log" (the same) or "maxlog"."""

    def __init__(self, encoder=None, gen_poly=None, rate=1 / 2, constraint_length=3, rsc=False, terminate=False,
                 hard_out=True, algorithm="map", precision=None, **kwargs):
        super().__init__(encoder, gen_poly, rate, constraint_length, rsc, terminate, precision, **kwargs)
        if algorithm not in ("map", "log", "maxlog"):
            raise ValueError("algorithm must be one of map, log or maxlog")
        if self._conv_k != 1:
            raise NotImplementedError("Only conv_k=1 currently supported.")
        self._hard_out = hard_out
        self._algorithm = algorithm

    def call(self, llr_ch, /, *, llr_a=None):
        y = self._rows(llr_ch)
        batch = y.shape[0]
        la = None
        if llr_a is not None:
            la = llr_a.to(device=y.device, dtype=torch.float32).reshape(batch, self._num_syms).contiguous()
        out = torch.empty((batch, self._k), dtype=torch.float32, device=y.device)
        ws = self._workspace(lib().sb_bcjr_workspace_bytes, batch, y.device)
        fr, op, ip = self._tables
        check(lib().sb_bcjr_decode(ptr(y), ptr(la), ptr(out), batch, self._num_syms, self._k,
                                   ("map", "log", "maxlog").index(self._algorithm), int(self._terminate),
                                   int(bool(self._hard_out)), ptr(fr), ptr(op), ptr(ip), self._ns, self._conv_n,
                                   ptr(ws), 0 if ws is None else ws.numel(), current_stream()), "sb_bcjr_decode")
        return out.to(self.rdtype).reshape(*llr_ch.shape[:-1], self._k)
