"""Interleavers (mirror of fec/interleaving.py:197-745): ``RandomInterleaver``, ``Deinterleaver`` and
``Turbo3GPPInterleaver``. A permutation is built on the host, kept on the device, and applied as one ``sb_gather_rows``
along the interleaved axis. ``RowColumnInterleaver`` and ``RandomInterleaver.find_s_min`` are not provided.

Deviations from the reference:
- Elements must be 4, 8 or 16 bytes wide (float32 / int32, float64 / int64 / complex64, complex128): the gather copies
  whole 32-bit words. Other dtypes raise ``TypeError``.
- ``RandomInterleaver`` draws its permutations from NumPy's generator, not from TensorFlow's ``stateless_uniform``; they
  are reproducible from ``seed`` (and from ``config.seed`` when no seed is given) but differ from the reference's."""
import numpy as np
import torch

from ..block import Block
from ..config import config
from ..._lib import lib, check, ptr, current_stream
from .qpp_table import QPP

_qpp = {K: (f1, f2) for K, f1, f2 in QPP}


def qpp_table():
    """TS 36.212 Table 5.1.3-3 as a dict K -> (f1, f2) (``qpp_table.py``, tools/make_turbo_tables.py)."""
    return _qpp


def turbo3gpp_perm(k):
    """int64 [k]: the QPP permutation pi(i) = (f1 i + f2 i^2) mod K of the smallest tabulated K >= k, with the entries
    >= k dropped (interleaving.py:678-712). k > 6144 raises ValueError."""
    tab = qpp_table()
    sizes = [K for K in tab if K >= k]
    if k < 1 or not sizes:
        raise ValueError("3GPP Turbo Interleaver is defined for block lengths up to 6144.")
    K = min(sizes)
    f1, f2 = tab[K]
    i = np.arange(K, dtype=np.int64)
    p = (f1 * i + f2 * i * i) % K
    return p[p < k]


def random_perms(seed, n, batch_size):
    """int64 [batch_size, n]: batch_size random permutations of 0 ... n - 1, a function of the integer seed only (NumPy's
    PCG64 seeded with (1337, seed), argsort of uniform draws as interleaving.py:387-393 does)."""
    rng = np.random.default_rng([1337, int(seed) & 0xFFFFFFFF])
    return np.argsort(rng.random((batch_size, n)), axis=-1, kind="stable")


def apply_perm(x, idx_dev, axis):
    """out = x gathered along `axis` by the int32 device index rows idx_dev: [n] (one permutation for all) or [B, n] (one
    per index of x's first dimension), out[..., j, ...] = x[..., idx[j], ...]; through ``sb_gather_rows``."""
    if x.element_size() not in (4, 8, 16) or x.dtype == torch.bool:
        raise TypeError(f"interleaving supports 4-, 8- and 16-byte elements, not {x.dtype}")
    xt = x.movedim(axis, -1).contiguous()
    n = xt.shape[-1]
    out = torch.empty_like(xt)
    if xt.numel() == 0:
        return out.movedim(-1, axis)
    words = x.element_size() // 4
    if idx_dev.dim() == 1:                               # one index row for every line
        batch, rows, in_rows = xt.numel() // n, 1, 1
    else:                                                # one index row per example, repeated over its lines
        per = xt.numel() // (n * idx_dev.shape[0])
        if per > 1:
            idx_dev = idx_dev.repeat_interleave(per, dim=0).contiguous()
        batch, rows, in_rows = 1, idx_dev.shape[0], idx_dev.shape[0]
    check(lib().sb_gather_rows(ptr(xt), ptr(idx_dev), ptr(out), batch, rows, n, in_rows, n, words, current_stream()),
          "sb_gather_rows")
    return out.movedim(-1, axis)


def _device_idx(p):
    return torch.from_numpy(np.ascontiguousarray(p, np.int32)).to(config.device)


class RandomInterleaver(Block):
    """RandomInterleaver(seed=None, keep_batch_constant=True, inverse=False, keep_state=True, axis=-1, precision=None)

    Random permutation of the entries of x along ``axis`` (interleaving.py:197-498). ``dec(x, seed=None, inverse=None)``.
    ``keep_state``: every call uses the permutation of ``seed`` (drawn from ``config``'s NumPy generator when not given);
    otherwise each call draws a new seed, and inverting then needs an explicit seed. ``keep_batch_constant=False``: one
    permutation per index of the first dimension. The permutations come from NumPy's generator, not TensorFlow's, so
    they are reproducible here but not equal to the reference's draws."""
    _native_double = True                                    # a pure copy: float64 stays float64

    def __init__(self, seed=None, keep_batch_constant=True, inverse=False, keep_state=True, axis=-1, precision=None,
                 **kwargs):
        super().__init__(precision=precision, **kwargs)
        if not isinstance(keep_batch_constant, bool):
            raise TypeError("keep_batch_constant must be bool.")
        self._keep_batch_constant = keep_batch_constant
        if not isinstance(axis, int):
            raise TypeError("axis must be int.")
        self._axis = axis
        if seed is not None:
            if not isinstance(seed, int):
                raise TypeError("seed must be int.")
        else:
            seed = int(config.np_rng.integers(0, 2 ** 31 - 1))
        self._seed = (1337, seed)
        if not isinstance(inverse, bool):
            raise TypeError("inverse must be boolean")
        self._inverse = inverse
        if not isinstance(keep_state, bool):
            raise TypeError("keep_state must be boolean")
        self._keep_state = keep_state
        if self._keep_state is False and self._inverse is True:
            print("Note: keep_state=False and, thus, a new realization of the interleaver is generated during each "
                  "call. Thus, the inverse interleaver does not correspond to a previous interleaver call.")
        self._cache = {}

    @property
    def seed(self):
        """Seed of the permutation used with ``keep_state``"""
        return self._seed[1]

    @property
    def axis(self):
        """Axis to be permuted"""
        return self._axis

    @property
    def keep_state(self):
        """Whether every call uses the permutation of ``seed``"""
        return self._keep_state

    def perm(self, n, seed=None, batch_size=1, inverse=False):
        """int64 [batch_size, n] host permutations of the given seed (default: this interleaver's)."""
        p = random_perms(self._seed[1] if seed is None else seed, n, batch_size)
        return np.argsort(p, axis=-1) if inverse else p

    def _perm_dev(self, seed, n, batch_size, inverse):
        key = (seed, n, batch_size, inverse, config.device)
        if key not in self._cache:
            if len(self._cache) > 8:
                self._cache.clear()
            p = self.perm(n, seed, batch_size, inverse)
            self._cache[key] = _device_idx(p[0] if self._keep_batch_constant or batch_size == 1 else p)
        return self._cache[key]

    def build(self, input_shape, **kwargs):
        if self._axis >= len(input_shape):
            raise ValueError("Axis does not match input shape.")

    def call(self, x, /, *, seed=None, inverse=None):
        if inverse is None:
            inverse = self._inverse
        elif not isinstance(inverse, bool):
            raise TypeError("inverse must be bool")
        if seed is not None:
            seed = int(seed)
        elif self._keep_state:
            seed = self._seed[1]
        else:
            if inverse:
                raise ValueError("Inverse interleaving not possible for random seeds per call (keep_state=False) "
                                 "without explicitly providing the seed as inputs.")
            seed = int(config.np_rng.integers(0, 2 ** 31 - 1))
        batch_size = 1 if self._keep_batch_constant or x.dim() == 1 else x.shape[0]
        idx = self._perm_dev(seed, x.shape[self._axis], batch_size, inverse)
        if batch_size > 1 and self._axis % x.dim() == 0:
            raise ValueError("Per-example permutations cannot permute the batch dimension.")
        return apply_perm(x, idx, self._axis)


class Turbo3GPPInterleaver(Block):
    """Turbo3GPPInterleaver(inverse=False, axis=-1, precision=None)

    The QPP interleaver of 3GPP turbo codes (TS 36.212 5.1.3.2.3, interleaving.py:598-745): x[..., pi(i), ...] moves to
    position i along ``axis``. For a length k that the table lacks, the next larger K is used and the entries >= k are
    dropped. Lengths above 6144 raise ``ValueError``."""
    _native_double = True

    def __init__(self, inverse=False, axis=-1, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if not isinstance(axis, int):
            raise TypeError("axis must be int.")
        self._axis = axis
        self._keep_state = True
        self.frame_size = None
        if not isinstance(inverse, bool):
            raise TypeError("inverse must be boolean")
        self._inverse = inverse
        self.coeffs_dict = qpp_table()
        self._cache = {}

    @property
    def axis(self):
        """Axis to be permuted"""
        return self._axis

    def perm(self, n, inverse=False):
        """int64 [n] host permutation (inverse: its inverse)."""
        p = turbo3gpp_perm(n)
        return np.argsort(p) if inverse else p

    def build(self, input_shape):
        if not self.axis < len(input_shape):
            raise ValueError("Axis does not match input shape.")
        if input_shape[self._axis] >= 6145:
            raise ValueError("3GPP Turbo Interleaver is defined for block lengths up to 6144.")

    def call(self, x, /, *, inverse=None, **kwargs):
        if inverse is None:
            inverse = self._inverse
        n = x.shape[self._axis]
        key = (n, inverse, config.device)
        if key not in self._cache:
            self._cache[key] = _device_idx(self.perm(n, inverse))
        return apply_perm(x, self._cache[key], self._axis)


class Deinterleaver(Block):
    """Deinterleaver(interleaver, precision=None)

    Reverts ``interleaver`` (interleaving.py:500-596): ``dec(x, seed=None)`` is ``interleaver(x, seed=seed,
    inverse=True)`` in x's dtype."""
    _native_double = True

    def __init__(self, interleaver, precision=None, **kwargs):
        if not isinstance(interleaver, (RandomInterleaver, Turbo3GPPInterleaver)):
            raise ValueError("interleaver is not a valid interleaver instance.")
        self._interleaver = interleaver
        if precision is None:
            precision = self._interleaver.precision
        super().__init__(precision=precision, **kwargs)
        if self._interleaver._keep_state is False:
            print("Warning: deinterleaver requires interleaver to have keep_state=True or to explicitly provide the "
                  "seed as inputs.")

    @property
    def interleaver(self):
        """Associated interleaver instance"""
        return self._interleaver

    def call(self, x, seed=None):
        return self._interleaver(x, seed=seed, inverse=True).to(x.dtype)
