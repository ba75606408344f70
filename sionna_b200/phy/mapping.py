"""Constellations, mapping and demapping (mirror of /root/reference/src/sionna/phy/mapping.py).

Host side: ``pam_gray`` / ``qam`` / ``pam`` (mapping.py:15-193) and ``Constellation`` (:195-469) build the point
tables with NumPy exactly as the reference does (38.211 5.1 Gray labelling, closed-form unit-energy
normalisation). Device side: ``Mapper`` -> ``sb_qam_map``, ``Demapper`` -> ``sb_demap``, ``SymbolDemapper`` ->
``sb_symbol_demap``, ``BinarySource`` -> ``sb_binary_source`` (``csrc/phy_kernels.cu``).
"""
import numpy as np
import torch

from .block import Block, Object  # noqa: F401
from .config import config, dtypes
from .._lib import lib, check, ptr, current_stream


def pam_gray(b):
    """Gray-labelled PAM point in {+-1, +-3, ...} for the bit vector ``b`` (recursion of 38.211 5.1, mapping.py:15-42)."""
    if len(b) > 1:
        return (1 - 2 * b[0]) * (2 ** len(b[1:]) - pam_gray(b[1:]))
    return 1 - 2 * b[0]


def qam(num_bits_per_symbol, normalize=True, precision=None):
    """QAM constellation; point ``n`` carries the binary label of ``n``, even bits -> real, odd bits -> imaginary
    PAM (mapping.py:44-118)."""
    try:
        assert num_bits_per_symbol % 2 == 0
        assert num_bits_per_symbol > 0
    except AssertionError as error:
        raise ValueError("num_bits_per_symbol must be a multiple of 2") from error
    assert isinstance(normalize, bool), "normalize must be boolean"
    prec = config.precision if precision is None else precision
    rdtype, cdtype = dtypes[prec]["np"]["rdtype"], dtypes[prec]["np"]["cdtype"]
    c = np.zeros([2 ** num_bits_per_symbol], dtype=cdtype)
    for i in range(2 ** num_bits_per_symbol):
        b = np.array(list(np.binary_repr(i, num_bits_per_symbol)), dtype=np.int32)
        c[i] = pam_gray(b[0::2]) + 1j * pam_gray(b[1::2])
    if normalize:
        n = int(num_bits_per_symbol / 2)
        qam_var = 1 / (2 ** (n - 2)) * np.sum(np.linspace(1, 2 ** n - 1, 2 ** (n - 1), dtype=rdtype) ** 2)
        c /= np.sqrt(qam_var)
    return c


def pam(num_bits_per_symbol, normalize=True, precision=None):
    """PAM constellation (real points in a complex array), mapping.py:120-193."""
    try:
        assert num_bits_per_symbol > 0
    except AssertionError as error:
        raise ValueError("num_bits_per_symbol must be positive") from error
    assert isinstance(normalize, bool), "normalize must be boolean"
    prec = config.precision if precision is None else precision
    rdtype, cdtype = dtypes[prec]["np"]["rdtype"], dtypes[prec]["np"]["cdtype"]
    c = np.zeros([2 ** num_bits_per_symbol], dtype=cdtype)
    for i in range(2 ** num_bits_per_symbol):
        b = np.array(list(np.binary_repr(i, num_bits_per_symbol)), dtype=np.int32)
        c[i] = pam_gray(b)
    if normalize:
        n = int(num_bits_per_symbol)
        pam_var = 1 / (2 ** (n - 1)) * np.sum(np.linspace(1, 2 ** n - 1, 2 ** (n - 1), dtype=rdtype) ** 2)
        c /= np.sqrt(pam_var)
    return c


class Constellation(Block):
    """Constellation(constellation_type, num_bits_per_symbol, points=None, normalize=False, center=False, precision=None)

    Vector of constellation points whose index is the bit label (mapping.py:195-469). ``call()`` returns the
    (possibly centred / normalised, for ``"custom"``) points as a complex tensor on the device."""

    def __init__(self, constellation_type, num_bits_per_symbol, points=None, normalize=False, center=False,
                 precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        if constellation_type not in ("qam", "pam", "custom"):
            raise ValueError(f"Wrong `constellation_type` {constellation_type}")
        self._constellation_type = constellation_type
        if num_bits_per_symbol is None:
            raise ValueError("No value for `num_bits_per_symbol`")
        n = num_bits_per_symbol
        if (n <= 0) or (n % 1 != 0):
            raise ValueError("`num_bits_per_symbol` must be a positive integer")
        if constellation_type == "qam" and n % 2 != 0:
            raise ValueError("`num_bits_per_symbol` must be a positive integer multiple of 2")
        self._num_bits_per_symbol = int(n)
        self._num_points = 2 ** self._num_bits_per_symbol
        self.normalize = normalize
        self.center = center
        if (points is not None) and (constellation_type != "custom"):
            raise ValueError("`points` can only be provided for `constellation_type`='custom'")
        if (points is None) and (constellation_type == "custom"):
            raise ValueError("You must provide a value for `points`")
        self._points = None
        if constellation_type == "qam":
            points = qam(self._num_bits_per_symbol, normalize=True, precision=precision)
        elif constellation_type == "pam":
            points = pam(self._num_bits_per_symbol, normalize=True, precision=precision)
        self.points = points
        self._dev_cache = None

    @property
    def constellation_type(self):
        return self._constellation_type

    @property
    def num_bits_per_symbol(self):
        return self._num_bits_per_symbol

    @property
    def num_points(self):
        return self._num_points

    @property
    def normalize(self):
        return self._normalize

    @normalize.setter
    def normalize(self, value):
        assert isinstance(value, bool), "`normalize` must be boolean"
        self._normalize = value
        self._dev_cache = None

    @property
    def center(self):
        return self._center

    @center.setter
    def center(self, value):
        assert isinstance(value, bool), "`center` must be boolean"
        self._center = value
        self._dev_cache = None

    @property
    def points(self):
        """[2**num_bits_per_symbol] complex points (host tensor; ``call()`` gives the device copy)."""
        return self._points

    @points.setter
    def points(self, v):
        if self._points is not None and self.constellation_type != "custom":
            raise ValueError("`points` can only be modified for custom constellations")
        v = torch.as_tensor(np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v))
        if tuple(v.shape) != (2 ** self.num_bits_per_symbol,):
            raise ValueError("`points` must have shape [2**num_bits_per_symbol]")
        self._points = v.to(self.cdtype)
        self._dev_cache = None

    def __call__(self):
        return self.call()

    def call(self):
        if self._dev_cache is None or self._dev_cache.device != self.device:
            x = self._points
            if self.constellation_type == "custom":
                if self._center:
                    x = x - x.mean()
                if self._normalize:
                    energy = (x.abs() ** 2).mean()
                    x = x / torch.sqrt(energy).to(x.dtype)
            self._dev_cache = x.to(self.device).contiguous()
        return self._dev_cache

    @staticmethod
    def check_or_create(*, constellation_type=None, num_bits_per_symbol=None, constellation=None, precision=None):
        """Return ``constellation`` if given, else build a "qam"/"pam" one (mapping.py:447-469)."""
        if isinstance(constellation, Constellation):
            return constellation
        if constellation_type in ["qam", "pam"]:
            return Constellation(constellation_type, num_bits_per_symbol, precision=precision)
        raise ValueError("You must provide a valid `constellation`")


def _need_single(obj, what):
    if obj.precision != "single":
        raise NotImplementedError(f"{what} is an fp32/complex64 kernel; precision='double' is not available.")


class Mapper(Block):
    """Mapper(constellation_type=None, num_bits_per_symbol=None, constellation=None, return_indices=False, precision=None)

    Maps ``[..., n]`` binary tensors to ``[..., n/num_bits_per_symbol]`` constellation points; within a symbol the
    first bit is the MSB of the point index (mapping.py:471-519)."""

    def __init__(self, constellation_type=None, num_bits_per_symbol=None, constellation=None, return_indices=False,
                 precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)
        self._return_indices = return_indices

    @property
    def constellation(self):
        return self._constellation

    def call(self, bits):
        _need_single(self, "sb_qam_map")
        m = self._constellation.num_bits_per_symbol
        bits = bits.to(device=self.device, dtype=torch.float32).contiguous()
        if bits.shape[-1] % m != 0:
            raise ValueError("The last input dimension must be a multiple of num_bits_per_symbol.")
        out_shape = list(bits.shape[:-1]) + [bits.shape[-1] // m]
        n_sym = bits.numel() // m
        pts = self._constellation().to(torch.complex64)          # the kernels read complex64 points
        x = torch.empty(out_shape, dtype=torch.complex64, device=self.device)
        idx = torch.empty(out_shape, dtype=torch.int32, device=self.device) if self._return_indices else None
        check(lib().sb_qam_map(ptr(bits), ptr(pts), m, ptr(x), ptr(idx), n_sym, current_stream()), "sb_qam_map")
        if self._return_indices:
            return x, idx
        return x


def _broadcast_inner(t, target_shape, device, dtype, trailing=0):
    """Return (contiguous tensor, inner) such that element ``s`` of the flattened target uses ``t_flat[s // inner]``.
    ``t`` must be broadcastable to ``target_shape`` after appending singleton dims (scalar, leading-dims-only and
    full-shape inputs avoid any materialisation)."""
    t = torch.as_tensor(t).to(device=device, dtype=dtype)
    tgt = list(target_shape)
    total = int(np.prod(tgt)) if tgt else 1
    if t.numel() == 1:
        return t.reshape(1).contiguous(), max(total, 1)
    shp = list(t.shape)
    while len(shp) < len(tgt):
        shp.append(1)
    t = t.reshape(shp)
    # leading-dims-only pattern: [d0, .., dk, 1, .., 1]
    k = len(shp)
    while k > 0 and shp[k - 1] == 1:
        k -= 1
    if shp[:k] == tgt[:k]:
        inner = int(np.prod(tgt[k:])) if k < len(tgt) else 1
        return t.reshape(-1).contiguous(), inner
    return t.expand(tgt).contiguous().reshape(-1), 1


def separable_levels_np(p, m):
    """(levels_re, levels_im) float32 arrays if every point of the 2^m-point constellation ``p`` equals
    levels_re[even label bits] + 1j * levels_im[odd label bits] exactly (all square QAMs, mapping.py:104-117), else None."""
    p = np.asarray(p)
    if m % 2 != 0 or not 2 <= m <= 10:
        return None
    h = m // 2
    j = np.arange(len(p))
    bits = (j[:, None] >> np.arange(m - 1, -1, -1)) & 1
    w = 1 << np.arange(h - 1, -1, -1)
    jr, ji = bits[:, 0::2] @ w, bits[:, 1::2] @ w
    lev_re, lev_im = np.zeros(1 << h, np.float32), np.zeros(1 << h, np.float32)
    lev_re[jr[ji == 0]] = p.real[ji == 0]
    lev_im[ji[jr == 0]] = p.imag[jr == 0]
    if np.array_equal(lev_re[jr], p.real.astype(np.float32)) and np.array_equal(lev_im[ji], p.imag.astype(np.float32)):
        return lev_re, lev_im
    return None


class Demapper(Block):
    """Demapper(demapping_method, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    LLRs (logits ``log p(b=1)/p(b=0)``) or hard decisions for received symbols ``y`` with noise variance ``no`` and
    optional bit priors (mapping.py:521-691, 794-967): ``"app"`` = log-sum-exp over the points with bit i = 1 minus
    the same over bit i = 0 of ``-|y-c|^2/no`` (+ log prior); ``"maxlog"`` replaces log-sum-exp by max."""

    def __init__(self, demapping_method, constellation_type=None, num_bits_per_symbol=None, constellation=None,
                 hard_out=False, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        assert demapping_method in ("app", "maxlog"), "Unknown demapping method"
        self._method = 0 if demapping_method == "app" else 1
        self._hard_out = hard_out
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)

    @property
    def constellation(self):
        return self._constellation

    def call(self, y, no, prior=None):
        _need_single(self, "sb_demap")
        m = self._constellation.num_bits_per_symbol
        dev = self.device
        y = y.to(device=dev, dtype=torch.complex64).contiguous()
        n_sym = y.numel()
        no_t, no_inner = _broadcast_inner(no, y.shape, dev, torch.float32)
        pr_t, pr_inner = None, 1
        if prior is not None:
            p = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if p.shape[-1] != m:
                raise ValueError("prior must have num_bits_per_symbol as last dimension.")
            if p.dim() == 1:
                pr_t, pr_inner = p.contiguous(), max(n_sym, 1)
            else:
                pr_t, pr_inner = p.expand(list(y.shape) + [m]).contiguous().reshape(-1), 1
        llr = torch.empty(list(y.shape[:-1]) + [y.shape[-1] * m], dtype=torch.float32, device=dev)
        pts = self._constellation().to(torch.complex64)          # the kernels read complex64 points
        levels = self._separable_levels(pts) if prior is None else None
        if levels is not None:                                  # square QAM: per-dimension kernel
            check(lib().sb_demap_qam(ptr(y), ptr(no_t), no_inner, ptr(levels[0]), ptr(levels[1]), m, self._method,
                                     ptr(llr), n_sym, int(self._hard_out), current_stream()), "sb_demap_qam")
            return llr
        check(lib().sb_demap(ptr(y), ptr(no_t), no_inner, ptr(pts), m, self._method, ptr(pr_t),
                             pr_inner, ptr(llr), n_sym, int(self._hard_out), current_stream()), "sb_demap")
        return llr

    def _separable_levels(self, pts):
        """Device tensors (levels_re, levels_im) if every point equals levels_re[even label bits] + 1j * levels_im[odd
        label bits] exactly (all square QAMs, mapping.py:104-117), else None. Cached per constellation tensor."""
        key = (pts.data_ptr(), pts._version, pts.device)
        if getattr(self, "_sep_key", None) == key:
            return self._sep_val
        lev = separable_levels_np(pts.detach().cpu().numpy(), self._constellation.num_bits_per_symbol)
        val = None if lev is None else (torch.from_numpy(lev[0]).to(pts.device), torch.from_numpy(lev[1]).to(pts.device))
        self._sep_key, self._sep_val = key, val
        return val


class SymbolDemapper(Block):
    """SymbolDemapper(constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False, precision=None)

    Normalised log-probabilities (logits) or hard decisions on the constellation points for received symbols
    (mapping.py:693-792): ``e_c = -|y - c|^2 / no + prior_c`` and ``log_softmax(e)`` over the points, or the index of
    the first maximum of ``e`` (``hard_out``). ``call(y [..., n], no, prior=None)``: ``no`` a scalar or broadcastable
    to ``y``, ``prior`` logits ``[num_points]`` or broadcastable to ``[..., n, num_points]`` -> ``[..., n, num_points]``
    float or ``[..., n]`` int32. Kernel: ``sb_symbol_demap``."""

    def __init__(self, constellation_type=None, num_bits_per_symbol=None, constellation=None, hard_out=False,
                 precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._hard_out = hard_out
        self._constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                            num_bits_per_symbol=num_bits_per_symbol,
                                                            constellation=constellation, precision=precision)

    @property
    def constellation(self):
        return self._constellation

    def call(self, y, no, prior=None):
        _need_single(self, "sb_symbol_demap")
        dev = self.device
        npts = self._constellation.num_points
        y = y.to(device=dev, dtype=torch.complex64).contiguous()
        n_sym = y.numel()
        no_t, no_inner = _broadcast_inner(no, y.shape, dev, torch.float32)
        pr_t, pr_inner = None, 1
        if prior is not None:
            p = torch.as_tensor(prior).to(device=dev, dtype=torch.float32)
            if p.dim() == 1:
                pr_t, pr_inner = p.expand(npts).contiguous(), max(n_sym, 1)
            else:
                pr_t = p.expand(list(y.shape) + [npts]).contiguous().reshape(-1)
        if self._hard_out:
            out = torch.empty(list(y.shape), dtype=torch.int32, device=dev)
        else:
            out = torch.empty(list(y.shape) + [npts], dtype=torch.float32, device=dev)
        pts = self._constellation().to(torch.complex64)
        check(lib().sb_symbol_demap(ptr(y), ptr(no_t), no_inner, ptr(pts), npts, ptr(pr_t), pr_inner, ptr(out), n_sym,
                                    int(bool(self._hard_out)), current_stream()), "sb_symbol_demap")
        return out


class BinarySource(Block):
    """BinarySource(precision=None, seed=None): random 0/1 tensor of the requested shape (mapping.py:1317-1352),
    drawn on the device with Philox4x32-10. ``seed`` gives the block its own stream; otherwise the global
    ``config`` stream is used."""

    def __init__(self, precision=None, seed=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        self._seed = seed
        self._offset = 0

    def __call__(self, inputs):
        return self._invoke(inputs)

    def call(self, inputs):
        shape = [int(s) for s in (inputs.tolist() if hasattr(inputs, "tolist") else inputs)]
        n = int(np.prod(shape)) if shape else 1
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        if self._seed is not None:
            seed, off = (int(self._seed) * 0x9E3779B97F4A7C15 + 0xABCDEF) & 0x7FFFFFFFFFFFFFFF, self._offset
            self._offset += 1
        else:
            seed, off = config.next_philox()
        check(lib().sb_binary_source(ptr(out), n, seed, off, current_stream()), "sb_binary_source")
        return out.to(self.rdtype)


class SymbolInds2Bits(Block):
    """SymbolInds2Bits(num_bits_per_symbol, precision=None): symbol indices -> their binary label, MSB first
    (mapping.py:1140-1179): ``[..., n]`` int -> ``[..., n, num_bits_per_symbol]`` float."""

    def __init__(self, num_bits_per_symbol, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        m = int(num_bits_per_symbol)
        labels = (np.arange(2 ** m)[:, None] >> np.arange(m - 1, -1, -1)) & 1
        self._labels_np = labels.astype(np.float32)
        self._labels = None

    def call(self, symbol_ind):
        ind = torch.as_tensor(symbol_ind).to(self.device).long()
        if self._labels is None or self._labels.device != ind.device:
            self._labels = torch.from_numpy(self._labels_np).to(ind.device)
        return self._labels[ind]


class SymbolSource(Block):
    """SymbolSource(constellation_type=None, num_bits_per_symbol=None, constellation=None, return_indices=False, return_bits=False, seed=None, precision=None)

    Random constellation symbols of the requested shape (mapping.py:1355-1445): `BinarySource` + `Mapper`. Returns
    ``symbols`` or ``[symbols, (indices), (bits)]``."""

    def __init__(self, constellation_type=None, num_bits_per_symbol=None, constellation=None, return_indices=False,
                 return_bits=False, seed=None, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)
        constellation = Constellation.check_or_create(constellation_type=constellation_type,
                                                      num_bits_per_symbol=num_bits_per_symbol,
                                                      constellation=constellation, precision=precision)
        self._num_bits_per_symbol = constellation.num_bits_per_symbol
        self._return_indices, self._return_bits = return_indices, return_bits
        self._binary_source = BinarySource(seed=seed, precision=precision)
        self._mapper = Mapper(constellation=constellation, return_indices=return_indices, precision=precision)

    def __call__(self, inputs):
        return self._invoke(inputs)

    def call(self, inputs):
        shape = [int(v) for v in (inputs.tolist() if hasattr(inputs, "tolist") else inputs)]
        b = self._binary_source(shape + [self._num_bits_per_symbol])
        if self._return_indices:
            x, ind = self._mapper(b)
        else:
            x = self._mapper(b)
        result = x.squeeze(-1)
        if self._return_indices or self._return_bits:
            result = [result]
        if self._return_indices:
            result.append(ind.squeeze(-1))
        if self._return_bits:
            result.append(b)
        return result


class QAMSource(SymbolSource):
    """QAMSource(num_bits_per_symbol=None, return_indices=False, return_bits=False, seed=None, precision=None) (mapping.py:1447-1500)."""

    def __init__(self, num_bits_per_symbol=None, return_indices=False, return_bits=False, seed=None, precision=None,
                 **kwargs):
        super().__init__(constellation_type="qam", num_bits_per_symbol=num_bits_per_symbol, return_indices=return_indices,
                         return_bits=return_bits, seed=seed, precision=precision, **kwargs)


class PAMSource(SymbolSource):
    """PAMSource(num_bits_per_symbol=None, return_indices=False, return_bits=False, seed=None, precision=None) (mapping.py:1502-1555)."""

    def __init__(self, num_bits_per_symbol=None, return_indices=False, return_bits=False, seed=None, precision=None,
                 **kwargs):
        super().__init__(constellation_type="pam", num_bits_per_symbol=num_bits_per_symbol, return_indices=return_indices,
                         return_bits=return_bits, seed=seed, precision=precision, **kwargs)
